// hqs_tick.cuh — tick_k: ONE cooperative kernel per scheduler tick.  Included by hqsched.cu inside its
// anonymous namespace (after hqs_ready_set.cuh and hqs_solver.cuh).
//
//   CTA 0 ("solver CTA")     stages the worker state, the class table and the tick's orders in shared memory
//                            (straight from the pinned host buffer, while the other CTAs count), waits for the
//                            histogram, compacts the non-empty (priority level, class) groups and then ONE warp
//                            walks them in priority order: a sparse first-fit over tiles of 32 workers (lane =
//                            worker) that starts at the class's frontier tile — the first tile that may still
//                            hold a worker with room for the class — so a group costs one or two tile visits
//                            instead of a block-wide scan.  The other 15 warps sleep on a named barrier and are
//                            woken for the block-parallel steps (quotas / capping of the packed level, restarts
//                            of the min-utilisation rule).
//   CTAs 1.. ("worker CTAs") count: per-chunk histogram of the ready tasks by group (4 B/slot streamed from HBM);
//                            scan:  exclusive prefix of the chunk table over chunks, one warp per group column;
//                            pack:  on request, one warp fills one worker (pack_body, the first saturated level);
//                            emit:  stable rank of every ready task inside its group -> count segment ->
//                                   (worker, variant), 8-byte assignment, READY -> DONE; the assignments of a chunk
//                                   are staged in shared memory and written as one contiguous run per group.
// Phases are ordered by acquire/release counters in global memory (TickSync); every wait has a time-out, so a
// broken grid fails the tick instead of hanging the GPU.  A sharded tick (several GPUs) exchanges the per-group
// counts by NVLink peer stores from the solver CTA between the histogram and the solve.
#pragma once

constexpr u32 TICK_THREADS = 512;
constexpr u32 TICK_WARPS = TICK_THREADS / 32;
constexpr u32 EMIT_ROWS_MAX = 20;     // rows of 32 tasks per emit warp and chunk (1.34 M table slots are one chunk per worker CTA on 132 SMs)
constexpr u32 EMIT_SEG_SMEM = 1024;   // count segments cached in shared memory by the emit step
constexpr u32 CMD_PACK = 1, CMD_EMIT = 2, CMD_EXIT = 3;      // grid commands: cmd word = (sequence << 2) | type
constexpr u32 BLK_PACK = 1, BLK_RESTART = 2, BLK_END = 3, BLK_PREFILL = 4, BLK_WIDE = 5;    // block commands inside the solver CTA
constexpr u32 TF_COUNT = 1, TF_EMIT = 2, TF_PACK = 4, TF_NO_REFRESH = 8, TF_NO_WIDE = 16;   // TF_NO_REFRESH / TF_NO_WIDE: measuring aids (HQS_DEBUG_NO_REFRESH, HQS_DEBUG_NO_WIDE)
constexpr u32 WIDE_MAX_GROUP = 0x03FFFFFFu;   // largest group the wide first-fit handles (32-bit prefix sums)
constexpr u32 SM_NONE = 0xFFFFFFFFu;
constexpr u32 GLIST_GLOBAL_WORDS = 4 * HQS_MAX_GROUPS;   // group list in global memory: glist [2][G], gcl [G], kk [G]
constexpr u32 PF_SEG_CAP = 1u << 18;  // prefill segments (eligible workers summed over classes) per tick
constexpr u32 MU_MAX_PASSES = 8;      // restarts of the min-utilisation rule before the remaining violators are dropped

struct TickSync {
    u32 cmd;          // grid command of the solver CTA
    u32 count_done;   // worker CTAs that finished their histograms
    u32 scan_done;    // worker CTAs that finished their part of the column scan
    u32 pack_done;    // worker CTAs that finished the current pack command (cumulative)
    u32 emit_done;    // worker CTAs that left the kernel's work loop
    u32 error;        // 2 = a wait timed out
    u32 pad[2];
#ifdef HQS_TRACE
    unsigned long long tr_emit[6];   // measuring build: %globaltimer maxima over the worker CTAs of the emit steps (TR_EMIT_*), CTAs with work
#endif
};
#ifdef HQS_TRACE
// emit steps of a worker CTA: command seen, group records + segments staged, chunk filter done, emit_finish done, emit_done counted
constexpr int TR_EMIT_CMD = 0, TR_EMIT_STAGED = 1, TR_EMIT_FILTER = 2, TR_EMIT_FINISH = 3, TR_EMIT_DONE = 4, TR_EMIT_NWORK = 5;
#define TR_EMIT(a, i) { if (threadIdx.x == 0) atomicMax(&(a).sync->tr_emit[i], global_timer_ns()); }
#else
#define TR_EMIT(a, i)
#endif

// offsets into the solver CTA's dynamic shared memory (SM_NONE: the array stays in global memory)
struct TickSmem {
    u32 fr, rem, unt, remtime, excl, touch, td, frontier, noresv; // always staged
    u32 glist, gcl;                                                // staged unless the mandatory arrays do not fit with them
    u32 classes, vorder, blocked, bef, loc;                        // optional
    u32 kk, top, pflvl;                                            // proactive filling only (kk: staged with glist)
};

struct TickArgs {
    // tick input: device-visible copy of the host staging buffer (pinned host memory read in place, or its device copy)
    const u64* free_rw;      // [W][R]
    const u64* total_rw;     // [W][R]
    const u64* rem_time;     // [W]
    const u32* order;        // [Q] class ids in processing order inside one priority level
    const uint8_t* vorder;   // [Q][HQS_MAX_VARIANTS] variant ids, first = the tick's demand variant
    const uint8_t* blocked;  // [W][Q] bytes (bit v) or nullptr
    const float* min_util;   // [W] or nullptr (no worker has a minimum utilisation)
    const void* classes;     // ClassT<RT, AT>[Q] of the solver's width
    const void* classes64;   // ClassT<RT, u64>[Q] (the pack warps work on exact amounts)
    u64 gscale[HQS_MAX_RESOURCES];   // narrow path: amount = scaled amount * gscale[r] (+ a per-worker remainder)
    u32 W, Q, L, R, G;
    u32 classes_bytes;       // Q * sizeof(ClassT<RT, AT>)
    u32 flags;               // TF_*
    u32 any_time_limit;      // some worker has a finite remaining time
    // task table / chunk geometry
    u32* key;
    u32 n_handles, chunk, rows, P, nbits, emit_warps, g_smem;
    u32 emit_stage;          // the finishing pass writes each chunk's assignments as per-group runs staged in shared memory
    // counts
    u32* total_local;        // [G] ready tasks of this rank per group (count step; zeroed at the end of the tick)
    const u32* total_ext;    // [G] counts summed over ranks, provided by the host (NCCL variant) or nullptr
    const u32* before_ext;   // [G] counts of lower ranks (NCCL variant) or nullptr
    u32* table;              // [P][G]
    // outputs
    GroupOut* gout;          // [G]
    u32* seg_cum;            // [SEG_CAP] inclusive end rank of the segment inside its group
    u32* seg_wv;             // [SEG_CAP] worker | variant << 16
    u64* free_after;         // [W][R] device copy
    TickHeaderOut* hdr;      // device copy
    TickHeaderOut* hdr_host; // pinned host mirror: header followed by free_after [W][R] (read by hqs_tick_fetch)
    hqs_assignment* out;
    u32 out_cap;
    u32* rem_scratch;        // [W][RT] u64 as u32 pairs: narrow remainders when they do not fit shared memory
    u32* glist_glob;         // [GLIST_GLOBAL_WORDS]: the group list when it does not fit shared memory (sm.glist == SM_NONE)
    // proactive filling (mapping.rs:156-230); pf_shift == 0: off.  With it on, every (level, class) splits into two groups,
    // waiting tasks first, prefilled ones second (take_tasks, taskqueue.rs:320-355): g = (level * Q + class) * 2 + prefilled
    u32 pf_shift, pf_reserve, pf_max;
    const uint8_t* prefilled_wc;   // [W][Q] nonzero: the worker holds a prefilled task of the class (host mirror), or nullptr
    uint4* gout2;            // [G] {end rank of the prefill range, offset of its records behind the assignments, first prefill segment, segments}
    u32* pf_cum;             // [PF_SEG_CAP] prefill segments: inclusive end rank inside the group
    u32* pf_wk;              //                                    worker
    // peer-to-peer count exchange (sharded tick without a host collective): x_world == 0 => off
    u32* x_peer[HQS_MAX_PEERS];   // base of every rank's exchange buffer (own included)
    u32* x_all;              // [G] out: sum over ranks
    u32* x_before;           // [G] out: sum over lower ranks
    u32 x_world, x_rank, x_seq;
    // synchronisation, pack
    TickSync* sync;
    PackScratch pk;
    uint8_t* excl_glob;      // [W] workers excluded by the min-utilisation rule (read by the pack warps)
    TickSmem sm;
    u32 smem_solver;         // bytes of the solver layout (debug)
};

__device__ __forceinline__ void bar_named(u32 id, u32 n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// thread 0 of a CTA: wait until *p >= target (counters restart at zero every tick)
__device__ __forceinline__ bool spin_until_ge(const u32* p, u32 target) {
    const long long t0 = clock64();
    while (ld_acquire(p) < target) {
        if (clock64() - t0 > SPIN_TIMEOUT_CYCLES) return false;
        __nanosleep(40);
    }
    return true;
}

__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// lanes of the warp holding the same group id, in constant time: one ballot per key bit (match.any
// iterates once per DISTINCT key, and a warp of 32 tasks holds ~30 distinct (level, class) keys)
__device__ __forceinline__ u32 same_key_lanes(u32 act, u32 g, u32 nbits) {
    u32 peers = act;
    for (u32 b = 0; b < nbits; ++b) {
        const u32 bit = (g >> b) & 1u;
        const u32 bal = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? bal : ~bal;
    }
    return peers;
}

// =================================================================================================
// worker CTAs
// =================================================================================================
// count: histogram of the ready tasks of chunk b by group -> table row b, totals.  4 B read per table slot.
__device__ void count_chunk(const TickArgs& a, u32 b, u32* s_hist) {
    const u32 G = a.G, Q = a.Q;
    for (u32 g = threadIdx.x; g < G; g += blockDim.x) s_hist[g] = 0;
    __syncthreads();
    const u32 base = b * a.chunk;
    const u32 end = min(base + a.chunk, a.n_handles);
    // chunk and base are multiples of 512 => 16-byte aligned uint4 loads; a ragged tail is scalar
    const u32 vec_end = base + ((end - base) & ~3u);
    for (u32 rowb = base; rowb < end; rowb += blockDim.x * 8) {
        // two independent 16-byte loads in flight per thread
        u32 k[8];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const u32 i = rowb + h * blockDim.x * 4 + threadIdx.x * 4;
            if (i + 4 <= vec_end) {
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(a.key + i));
                k[4 * h] = v.x; k[4 * h + 1] = v.y; k[4 * h + 2] = v.z; k[4 * h + 3] = v.w;
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) k[4 * h + j] = (i + j < end) ? __ldg(a.key + i + j) : 0u;
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            // keys inside one warp are mostly distinct (levels x classes), so plain shared-memory atomics
            // beat warp aggregation (match.any costs one round per distinct key)
            if (k[j] & KEY_READY) atomicAdd(&s_hist[((key_level(k[j]) * Q + key_class(k[j])) << a.pf_shift) | ((k[j] >> 28) & a.pf_shift)], 1u);
        }
    }
    __syncthreads();
    u32* row = a.table + (size_t)b * G;
    for (u32 g = threadIdx.x; g < G; g += blockDim.x) {
        const u32 v = s_hist[g];
        row[g] = v;
        if (v) atomicAdd(&a.total_local[g], v);
    }
    __syncthreads();
}

// emit: stable (handle-ordered) rank of every ready task of chunk b inside its group, rank -> placement.
// Each warp owns a.rows rows of 32 consecutive tasks; per-warp group counters live in shared memory:
//   s_cnt[w][g]  first pass: tasks of group g in warp w's rows; then the rank at which warp w's first task of
//                group g starts; second pass: running counter.
// HBM traffic: 4 B read per table slot (L2 hit: the count step read it microseconds ago), 8 B written per
// assignment, 4 B key write-back per assignment.
// Two halves: emit_prepare needs the task table and the scanned chunk table only — a worker CTA with a single chunk
// runs it WHILE the solver CTA solves and keeps its rows in registers; emit_finish needs the solver's group records.
struct EmitRows { u32 kk[EMIT_ROWS_MAX], peers[EMIT_ROWS_MAX]; };

// the emit step's shared memory (worker CTAs)
struct EmitSmem {
    u32* cnt;              // [emit_warps][G] per-warp group counters
    GroupOut* go;          // [G] the solver's group records (g_smem)
    u32 *segc, *segw;      // [EMIT_SEG_SMEM] count segment cache
    uint4* run;            // [G + 1] per-group runs of the chunk (emit_stage)
    u32* slot;             // [chunk] staged tasks in run order (emit_stage)
    unsigned short* q;     // [chunk] place of each task in its run (emit_stage)
};

__device__ __forceinline__ EmitSmem emit_smem(const TickArgs& a, unsigned char* smem) {
    EmitSmem es;
    es.cnt = reinterpret_cast<u32*>(smem);
    es.go = reinterpret_cast<GroupOut*>(es.cnt + a.emit_warps * a.G);
    es.segc = reinterpret_cast<u32*>(es.go + (a.g_smem ? a.G : 0));
    es.segw = es.segc + EMIT_SEG_SMEM;
    es.run = reinterpret_cast<uint4*>(reinterpret_cast<uintptr_t>(es.segw + EMIT_SEG_SMEM + 3) & ~(uintptr_t)15);   // 16-byte aligned
    es.slot = reinterpret_cast<u32*>(es.run + a.G + 1);
    es.q = reinterpret_cast<unsigned short*>(es.slot + a.chunk);
    return es;
}

__device__ __forceinline__ void emit_stage_ranks(const TickArgs& a, u32 b, const EmitSmem& es, const EmitRows& er);

__device__ __forceinline__ void emit_prepare(const TickArgs& a, u32 b, const EmitSmem& es, EmitRows& er) {
    u32* s_cnt = es.cnt;
    const u32 G = a.G, Q = a.Q, nwarps = a.emit_warps, rows = a.rows;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u32* row = a.table + (size_t)b * G;
    for (u32 i = threadIdx.x; i < nwarps * G; i += blockDim.x) s_cnt[i] = 0;
    __syncthreads();
    const u32 base = b * a.chunk;
    const u32 end = min(base + a.chunk, a.n_handles);
    const bool active = warp < nwarps;
    const u32 wbeg = base + warp * (32 * rows);
    u32* mycnt = s_cnt + (active ? warp : 0) * G;
#pragma unroll
    for (int j = 0; j < (int)EMIT_ROWS_MAX; ++j) {
        const u32 i = wbeg + j * 32 + lane;
        er.kk[j] = (active && j < (int)rows && i < end) ? a.key[i] : 0u;
    }
#pragma unroll
    for (int j = 0; j < (int)EMIT_ROWS_MAX; ++j) {
        er.peers[j] = 0;
        if (active && j < (int)rows) {                       // warp-uniform
            const bool ready = (er.kk[j] & KEY_READY) != 0;
            const u32 g = ((key_level(er.kk[j]) * Q + key_class(er.kk[j])) << a.pf_shift) | ((er.kk[j] >> 28) & a.pf_shift);
            const u32 act = __ballot_sync(0xffffffffu, ready);
            u32 pm = same_key_lanes(act, g, a.nbits);
            if (!ready) pm = 0;
            er.peers[j] = pm;
            // pass 1: per-warp counts (rows in order; the leader of each key adds its lanes)
            if (ready && (u32)(__ffs(pm) - 1) == lane) mycnt[g] += __popc(pm);
            __syncwarp();
        }
    }
    __syncthreads();
    // turn counts into starting ranks: rank0(w, g) = table[b][g] + sum_{w' < w} cnt[w'][g]
    for (u32 g = threadIdx.x; g < G; g += blockDim.x) {
        const u32 first = __ldcg(row + g);
        u32 run = first;
        for (u32 w2 = 0; w2 < nwarps; ++w2) {
            const u32 c = s_cnt[w2 * G + g];
            s_cnt[w2 * G + g] = run;
            run += c;
        }
        if (a.emit_stage) es.run[g] = make_uint4(first, run - first, 0, 0);
    }
    __syncthreads();
    if (a.emit_stage) emit_stage_ranks(a, b, es, er);
}

// A chunk holds an assigned task only if, for some group, fewer than k[g] tasks of the group precede the chunk (the
// assigned ones are the first k[g] in handle order): in a drain tick only the first chunks qualify, the rest leave
// after reading one table row.
__device__ __forceinline__ bool emit_chunk_has_work(const TickArgs& a, u32 b, const GroupOut* s_go, const u32* before) {
    const u32 G = a.G;
    const u32* row = a.table + (size_t)b * G;
    bool mine = false;
    for (u32 g = threadIdx.x; g < G; g += blockDim.x) {
        const u32 bef = before ? __ldcg(before + g) : 0u;
        u32 k = a.g_smem ? s_go[g].k : __ldcg(&a.gout[g].k);
        if (a.pf_shift) { const u32 kpf = __ldcg(&a.gout2[g].x); k = k > kpf ? k : kpf; }      // the prefill range lies behind the assigned ranks
        mine |= __ldcg(row + g) + bef < k;
    }
    return __syncthreads_or(mine) != 0;
}

__device__ __forceinline__ void emit_finish(const TickArgs& a, u32 b, u32* s_cnt, const GroupOut* s_go, const u32* s_segc, const u32* s_segw,
                                            bool seg_smem, const u32* before, u32 n_assigned, const EmitRows& er) {
    const u32 G = a.G, Q = a.Q, nwarps = a.emit_warps, rows = a.rows;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u32 base = b * a.chunk;
    const bool active = warp < nwarps;
    const u32 wbeg = base + warp * (32 * rows);
    u32* mycnt = s_cnt + (active ? warp : 0) * G;
    // pass 2: rank and emit
#pragma unroll
    for (int j = 0; j < (int)EMIT_ROWS_MAX; ++j) {
        if (active && j < (int)rows) {                       // warp-uniform
            const u32 i = wbeg + j * 32 + lane;
            const u32 k = er.kk[j], pm = er.peers[j];
            const u32 g = ((key_level(k) * Q + key_class(k)) << a.pf_shift) | ((k >> 28) & a.pf_shift);
            if (pm) {
                const u32 leader = __ffs(pm) - 1;
                u32 r0 = 0;
                if (leader == lane) {
                    r0 = mycnt[g];
                    mycnt[g] = r0 + __popc(pm);
                }
                r0 = __shfl_sync(pm, r0, leader);
                const u32 r_loc = r0 + __popc(pm & ((1u << lane) - 1));      // rank among this rank's tasks
                const u32 bef = before ? __ldcg(before + g) : 0u;
                GroupOut go;
                if (a.g_smem) go = s_go[g];
                else {
                    const uint4 gv = __ldcg(reinterpret_cast<const uint4*>(a.gout + g));
                    go.k = gv.x; go.out_off = gv.y; go.seg_lo = gv.z; go.seg_n = gv.w;
                }
                if (r_loc + bef < go.k) {
                    const u32 r = r_loc + bef;                                // global rank in the group
                    // first segment whose inclusive end rank exceeds r
                    u32 lo = go.seg_lo, hi = go.seg_lo + go.seg_n;
                    u32 wv;
                    if (seg_smem) {
                        while (lo < hi) {
                            const u32 mid = (lo + hi) >> 1;
                            if (s_segc[mid] > r) hi = mid; else lo = mid + 1;
                        }
                        wv = s_segw[lo];
                    } else {
                        while (lo < hi) {
                            const u32 mid = (lo + hi) >> 1;
                            if (__ldcg(a.seg_cum + mid) > r) hi = mid; else lo = mid + 1;
                        }
                        wv = __ldcg(a.seg_wv + lo);
                    }
                    const u32 oi = go.out_off + r_loc;
                    if (oi < a.out_cap) {
                        hqs_assignment asg;
                        asg.task = i;
                        asg.worker = (uint16_t)(wv & 0xFFFFu);
                        asg.variant = (uint8_t)((wv >> 16) & 0xFFu);
                        asg.kind = (k & KEY_PF) ? 2 : 0;                      // a prefilled task: retract + redirect (mapping.rs:63-101)
                        a.out[oi] = asg;
                        a.key[i] = (k & ~(KEY_READY | KEY_PF)) | KEY_DONE;    // Waiting / Prefilled -> Assigned / Retracting
                    }
                } else if (a.pf_shift && !(k & KEY_PF)) {
                    // proactive filling: the waiting tasks right behind the assigned ones go to the workers that just
                    // received tasks of the class; they stay ready
                    const uint4 g2 = __ldcg(a.gout2 + g);
                    if (r_loc + bef < g2.x) {
                        const u32 r = r_loc + bef;
                        u32 lo = g2.z, hi = g2.z + g2.w;
                        while (lo < hi) {
                            const u32 mid = (lo + hi) >> 1;
                            if (__ldcg(a.pf_cum + mid) > r) hi = mid; else lo = mid + 1;
                        }
                        const u32 oi = n_assigned + g2.y + (r - max(go.k, bef));      // sharded: this rank's part of the range
                        if (oi < a.out_cap) {
                            hqs_assignment asg;
                            asg.task = i;
                            asg.worker = (uint16_t)__ldcg(a.pf_wk + lo);
                            asg.variant = 0xFF;                                   // ComputeTasks with variant = None
                            asg.kind = 1;
                            a.out[oi] = asg;
                            a.key[i] = k | KEY_PF;
                        }
                    }
                }
            }
            __syncwarp();
        }
    }
    __syncthreads();
}

// Finishing pass on per-group runs (a.emit_stage).  The ready tasks of group g in chunk b have the consecutive local ranks
// table[b][g] ... table[b][g] + cnt_b[g] - 1, and the assigned ones are the first n_b[g] of them, so the chunk's records form
// ONE contiguous run of the output per group, starting at out_off[g] + table[b][g].  emit_stage_ranks (part of emit_prepare,
// i.e. while the solver CTA still solves) writes every ready task to a shared-memory slot at its run's base + its place in
// the run (bases: exclusive prefix of cnt_b over the groups) and remembers that place per task.  Once the group records
// are out, emit_finish_staged writes the keys back row by row and flushes the slots in order, a thread per slot, so a warp
// stores 32 consecutive records of a run instead of ~30 scattered ones.  A tick with a prefill range (kind-1 records
// behind the assigned ranks) takes the per-task pass (emit_finish) on the same prepared rows.
// Slot word: task offset inside the chunk (15 bits) | prefilled << 15 | group << 16.
constexpr u32 STAGE_OFF_MASK = 0x7FFFu, STAGE_PF = 1u << 15, STAGE_G_SHIFT = 16;
static_assert(TICK_THREADS * EMIT_ROWS_MAX <= STAGE_OFF_MASK + 1 && 2 * HQS_MAX_GROUPS <= (1u << (32 - STAGE_G_SHIFT)), "slot word");

__device__ __forceinline__ void emit_stage_ranks(const TickArgs& a, u32 b, const EmitSmem& es, const EmitRows& er) {
    __shared__ u32 s_wsum[TICK_WARPS];
    const u32 G = a.G, Q = a.Q, nwarps = a.emit_warps, rows = a.rows;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u32 base = b * a.chunk;
    // es.run[g] = {table[b][g], cnt_b[g], slot base} (emit_prepare wrote the first two); a thread owns `per` consecutive
    // groups, the slot bases are a block-wide exclusive prefix; es.run[G].x = ready tasks of the chunk
    const u32 per = (G + blockDim.x - 1) / blockDim.x, g0 = min(threadIdx.x * per, G), g1 = min(g0 + per, G);
    u32 sum = 0;
    for (u32 g = g0; g < g1; ++g) { const u32 c = es.run[g].y; es.run[g].z = sum; sum += c; }
    u32 inc = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u32 y = __shfl_up_sync(0xffffffffu, inc, d);
        if ((int)lane >= d) inc += y;
    }
    if (lane == 31) s_wsum[warp] = inc;
    __syncthreads();
    u32 wbase = 0, n_ready = 0;
    for (u32 w2 = 0; w2 < TICK_WARPS; ++w2) { const u32 v = s_wsum[w2]; wbase += w2 < warp ? v : 0u; n_ready += v; }
    const u32 tbase = wbase + inc - sum;
    for (u32 g = g0; g < g1; ++g) es.run[g].z += tbase;
    if (threadIdx.x == 0) es.run[G] = make_uint4(n_ready, 0, 0, 0);
    __syncthreads();
    // ranks: the per-warp counters of emit_prepare, rows in order
    const bool active = warp < nwarps;
    const u32 wbeg = base + warp * (32 * rows);
    u32* mycnt = es.cnt + (active ? warp : 0) * G;
#pragma unroll
    for (int j = 0; j < (int)EMIT_ROWS_MAX; ++j) {
        if (active && j < (int)rows) {                       // warp-uniform
            const u32 k = er.kk[j], pm = er.peers[j];
            const u32 g = ((key_level(k) * Q + key_class(k)) << a.pf_shift) | ((k >> 28) & a.pf_shift);
            if (pm) {
                const u32 leader = __ffs(pm) - 1;
                u32 r0 = 0;
                if (leader == lane) {
                    r0 = mycnt[g];
                    mycnt[g] = r0 + __popc(pm);
                }
                r0 = __shfl_sync(pm, r0, leader);
                const uint4 run = es.run[g];
                const u32 q = r0 + __popc(pm & ((1u << lane) - 1)) - run.x;      // place in the chunk's run of the group
                const u32 off = wbeg + j * 32 + lane - base;
                es.slot[run.z + q] = off | ((k & KEY_PF) ? STAGE_PF : 0u) | (g << STAGE_G_SHIFT);
                es.q[off] = (unsigned short)q;
            }
            __syncwarp();
        }
    }
    __syncthreads();
    // the counters back to the warps' starting ranks (the per-task pass reads them): warp w's counter now holds warp w+1's
    for (u32 g = threadIdx.x; g < G; g += blockDim.x) {
        for (u32 w2 = nwarps - 1; w2 > 0; --w2) es.cnt[w2 * G + g] = es.cnt[(w2 - 1) * G + g];
        es.cnt[g] = es.run[g].x;
    }
    __syncthreads();
}

__device__ __forceinline__ void emit_finish_staged(const TickArgs& a, u32 b, const EmitSmem& es, bool seg_smem, const u32* before,
                                                   const EmitRows& er) {
    const u32 G = a.G, Q = a.Q, nwarps = a.emit_warps, rows = a.rows;
    const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 base = b * a.chunk;
    const u32 n_ready = es.run[G].x;
    // runs: es.run[g].y = assigned tasks (the first k[g] - before[g] - table[b][g] ranks, clamped to the run), .w = output
    // index of the run's first record
    for (u32 g = threadIdx.x; g < G; g += blockDim.x) {
        const uint4 run = es.run[g];
        const u32 bef = before ? __ldcg(before + g) : 0u;
        const GroupOut go = es.go[g];
        const u32 n = go.k > bef + run.x ? go.k - bef - run.x : 0u;
        es.run[g].y = n < run.y ? n : run.y;
        es.run[g].w = go.out_off + run.x;
    }
    __syncthreads();
    // keys, row by row (coalesced): Waiting / Prefilled -> Assigned / Retracting
    const bool active = warp < nwarps;
    const u32 wbeg = base + warp * (32 * rows);
#pragma unroll
    for (int j = 0; j < (int)EMIT_ROWS_MAX; ++j) {
        if (active && j < (int)rows && er.peers[j]) {
            const u32 k = er.kk[j];
            const u32 g = ((key_level(k) * Q + key_class(k)) << a.pf_shift) | ((k >> 28) & a.pf_shift);
            const u32 i = wbeg + j * 32 + lane;
            const u32 q = es.q[i - base];
            const uint4 run = es.run[g];
            if (q < run.y && run.w + q < a.out_cap) a.key[i] = (k & ~(KEY_READY | KEY_PF)) | KEY_DONE;
        }
    }
    // flush: slot s is record run.w + (s - run.z) of its group's run when s - run.z < run.y
    for (u32 s = threadIdx.x; s < n_ready; s += blockDim.x) {
        const u32 v = es.slot[s];
        const u32 g = v >> STAGE_G_SHIFT;
        const uint4 run = es.run[g];
        const u32 q = s - run.z;
        if (q >= run.y) continue;
        const u32 oi = run.w + q;
        if (oi >= a.out_cap) continue;
        const u32 r = run.x + q + (before ? __ldcg(before + g) : 0u);       // global rank in the group
        const GroupOut go = es.go[g];
        // first segment whose inclusive end rank exceeds r
        u32 lo = go.seg_lo, hi = go.seg_lo + go.seg_n;
        u32 wv;
        if (seg_smem) {
            while (lo < hi) {
                const u32 mid = (lo + hi) >> 1;
                if (es.segc[mid] > r) hi = mid; else lo = mid + 1;
            }
            wv = es.segw[lo];
        } else {
            while (lo < hi) {
                const u32 mid = (lo + hi) >> 1;
                if (__ldcg(a.seg_cum + mid) > r) hi = mid; else lo = mid + 1;
            }
            wv = __ldcg(a.seg_wv + lo);
        }
        // one 8-byte store: task | worker << 32 | variant << 48 | kind << 56 (hqs_assignment)
        const u32 hi_word = (wv & 0xFFFFu) | (((wv >> 16) & 0xFFu) << 16) | ((v & STAGE_PF) ? 2u << 24 : 0u);
        reinterpret_cast<uint2*>(a.out)[oi] = make_uint2(base + (v & STAGE_OFF_MASK), hi_word);
    }
    __syncthreads();
}

template <int RT>
__device__ void worker_cta(const TickArgs& a, unsigned char* smem) {
    __shared__ u32 s_cmd, s_ok;
    u32* s_u32 = reinterpret_cast<u32*>(smem);
    const u32 nW = gridDim.x - 1, me = blockIdx.x - 1;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    bool ok = true;
    // ---- count
    if (a.flags & TF_COUNT) {
        for (u32 b = me; b < a.P; b += nW) count_chunk(a, b, s_u32);
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            atomicAdd(&a.sync->count_done, 1u);
            s_ok = spin_until_ge(&a.sync->count_done, nW) ? 1u : 0u;
        }
        __syncthreads();
        ok = s_ok != 0;
    }
    // ---- scan: exclusive prefix over chunks, one warp per group column, 32 chunk rows per step
    if (ok) {
        for (u32 g = me * TICK_WARPS + warp; g < a.G; g += nW * TICK_WARPS) {
            u32 carry = 0;
            for (u32 b0 = 0; b0 < a.P; b0 += 32) {
                const u32 b = b0 + lane;
                const u32 v = b < a.P ? __ldcg(a.table + (size_t)b * a.G + g) : 0;
                u32 inc = v;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const u32 y = __shfl_up_sync(0xffffffffu, inc, d);
                    if ((int)lane >= d) inc += y;
                }
                if (b < a.P) a.table[(size_t)b * a.G + g] = carry + inc - v;
                carry += __shfl_sync(0xffffffffu, inc, 31);
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(&a.sync->scan_done, 1u);
    }
    // ---- first half of emit, while the solver CTA solves: a CTA that owns a single chunk ranks its ready tasks now and
    //      keeps the rows in registers (a pack command in between reuses the shared memory: then emit starts over)
    EmitRows er;
    bool prepared = false;
    if (ok && (a.flags & TF_EMIT) && me < a.P && a.P <= nW) {
        if (threadIdx.x == 0) s_ok = spin_until_ge(&a.sync->scan_done, nW) ? 1u : 0u;
        __syncthreads();
        prepared = s_ok != 0;
        __syncthreads();
        if (prepared) emit_prepare(a, me, emit_smem(a, smem), er);
    }
    // ---- command loop
    auto next_cmd = [&](u32 seen) -> u32 {
        if (threadIdx.x == 0) {
            u32 cmd = 0;
            if (ok) {
                const long long t0 = clock64();
                const long long limit = a.x_world ? PEER_TIMEOUT_CYCLES + SPIN_TIMEOUT_CYCLES : SPIN_TIMEOUT_CYCLES;
                while ((cmd = ld_acquire(&a.sync->cmd)) == seen) {
                    if (clock64() - t0 > limit) { cmd = 0; break; }
                    __nanosleep(100);
                }
            }
            if (cmd == 0 || cmd == seen) { atomicExch(&a.sync->error, 2u); cmd = CMD_EXIT; }
            s_cmd = cmd;
        }
        __syncthreads();
        const u32 cmd = s_cmd;
        __syncthreads();
        return cmd;
    };
    // emit of this CTA's chunks; rows != nullptr: chunk `me` was prepared above
    auto do_emit = [&](EmitRows* rows) {
        TR_EMIT(a, TR_EMIT_CMD)
        if (threadIdx.x == 0) s_ok = spin_until_ge(&a.sync->scan_done, nW) ? 1u : 0u;
        __syncthreads();
        if (s_ok) {
            const u32 G = a.G;
            const EmitSmem es = emit_smem(a, smem);
            GroupOut* s_go = es.go;                                                  // [G] when g_smem
            const u32 n_seg = __ldcg(&a.hdr->n_segments);
            const bool seg_smem = n_seg <= EMIT_SEG_SMEM;
            const u32* before = a.x_world ? a.x_before : a.before_ext;
            if (me < a.P) {
                if (a.g_smem)
                    for (u32 g = threadIdx.x; g < G; g += blockDim.x) {
                        const uint4 v = __ldcg(reinterpret_cast<const uint4*>(a.gout + g));
                        GroupOut go; go.k = v.x; go.out_off = v.y; go.seg_lo = v.z; go.seg_n = v.w;
                        s_go[g] = go;
                    }
                if (seg_smem)
                    for (u32 i = threadIdx.x; i < n_seg; i += blockDim.x) { es.segc[i] = __ldcg(a.seg_cum + i); es.segw[i] = __ldcg(a.seg_wv + i); }
                __syncthreads();
                TR_EMIT(a, TR_EMIT_STAGED)
                const u32 n_assigned = __ldcg(&a.hdr->n_assigned);
                // kind-1 records of a prefill range lie behind the assigned ranks: such a tick keeps the per-task pass (in a
                // sharded tick n_prefilled is this rank's, so a rank without prefill records may stage while its peers do not)
                const bool staged = a.emit_stage && __ldcg(&a.hdr->n_prefilled) == 0;
                auto finish = [&](u32 b, const EmitRows& r) {
                    if (staged) emit_finish_staged(a, b, es, seg_smem, before, r);
                    else emit_finish(a, b, es.cnt, s_go, es.segc, es.segw, seg_smem, before, n_assigned, r);
                };
                if (rows) {
                    const bool work = emit_chunk_has_work(a, me, s_go, before);
                    TR_EMIT(a, TR_EMIT_FILTER)
                    if (work) {
#ifdef HQS_TRACE
                        if (threadIdx.x == 0) atomicAdd(&a.sync->tr_emit[TR_EMIT_NWORK], 1ull);
#endif
                        finish(me, *rows);
                    }
                } else {
                    for (u32 b = me; b < a.P; b += nW) {
                        if (!emit_chunk_has_work(a, b, s_go, before)) continue;
                        EmitRows r2;
                        emit_prepare(a, b, es, r2);
                        finish(b, r2);
                    }
                    TR_EMIT(a, TR_EMIT_FILTER)
                }
                TR_EMIT(a, TR_EMIT_FINISH)
            }
        } else if (threadIdx.x == 0) {
            atomicExch(&a.sync->error, 2u);
        }
    };
    u32 cmd = next_cmd(0);
    if (prepared && (cmd & 3u) == CMD_EMIT) {
        do_emit(&er);                       // the prepared rows are used by the FIRST command only (a pack reuses the shared memory)
    } else {
        for (;;) {
            const u32 type = cmd & 3u;
            if (type == CMD_PACK) {
                PackArgs p;
                p.pk = a.pk; p.total_rw = a.total_rw; p.rem_time = a.rem_time; p.blocked = a.blocked;
                p.excluded = a.min_util ? a.excl_glob : nullptr; p.classes64 = a.classes64; p.W = a.W; p.Q = a.Q; p.R = a.R;
                pack_body<RT>(p, smem);
                __threadfence();
                __syncthreads();
                if (threadIdx.x == 0) atomicAdd(&a.sync->pack_done, 1u);
                cmd = next_cmd(cmd);
                continue;
            }
            if (type == CMD_EMIT) do_emit(nullptr);
            break;      // CMD_EMIT or CMD_EXIT
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        TR_EMIT(a, TR_EMIT_DONE)
        atomicAdd(&a.sync->emit_done, 1u);
    }
}

// =================================================================================================
// solver CTA
// =================================================================================================
template <int RT, typename AT>
__device__ void solver_cta(const TickArgs& a, unsigned char* smem) {
    constexpr bool NARROW = sizeof(AT) == 4;
    constexpr AT AMAX = AmountMax<AT>::value;
    using Var = VarT<RT, AT>;
    using Cls = ClassT<RT, AT>;
    __shared__ u64 s_C[HQS_MAX_RESOURCES], s_totmax[HQS_MAX_RESOURCES], s_D[HQS_MAX_RESOURCES];
    __shared__ u64 s_red[TICK_WARPS * (HQS_MAX_RESOURCES + 1)];
    __shared__ u64 s_qT[PACK_MAX_CAND];
    __shared__ u32 s_wcnt[TICK_WARPS];
    __shared__ u32 s_pkpos[PACK_MAX_CAND], s_pknseg[PACK_MAX_CAND], s_pkseglo[PACK_MAX_CAND], s_pkex[PACK_MAX_CAND], s_cbase[PACK_MAX_CAND + 1];
    __shared__ u32 s_blk[8];            // block command: type, li, lj, seg region base, phi (2 words), n_packs
    __shared__ u32 s_nlist, s_multi, s_err, s_final_err, s_npacks, s_partial, s_npref, s_bign;
    __shared__ u32 s_xmis;              // sharded tick: 1 << 31 | peer << 16 | the peer's G if a peer's group count differs
    __shared__ unsigned long long s_wx[2][TICK_WARPS];   // wide first-fit: one record per warp and group (double-buffered)
#ifdef HQS_TRACE
    __shared__ u32 s_trw[8];
    __shared__ unsigned long long s_trel;                // %globaltimer at the release of the grid's last command
#endif
    __shared__ u32 s_wc[TICK_WARPS];                     //                 per warp: count segments written for the LAST group
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 W = a.W, Q = a.Q, R = a.R, G = a.G;
    const u32 nW = gridDim.x - 1;
    const u32 n_tiles = (W + 31) / 32;
    const long long t_start = clock64();
    const unsigned long long gt_start = global_timer_ns();

    // ---- shared-memory layout
    AT* s_fr = reinterpret_cast<AT*>(smem + a.sm.fr);                                  // [W][RT]
    u32* s_unt = reinterpret_cast<u32*>(smem + a.sm.unt);                              // [W] bit r: free == total != 0
    u64* s_remtime = reinterpret_cast<u64*>(smem + a.sm.remtime);                      // [W]
    uint8_t* s_excl = smem + a.sm.excl;                                                // [W] 1: minimum utilisation, 2: reserved
    uint8_t* s_touch = smem + a.sm.touch;                                              // [W] the worker received something in this tick
    uint8_t* s_noresv = smem + a.sm.noresv;                                            // [Q] no worker can be reserved for the class any more
    unsigned short* s_td = reinterpret_cast<unsigned short*>(smem + a.sm.td);          // [W] tried | dead << 8 of the current group
    unsigned short* s_front = reinterpret_cast<unsigned short*>(smem + a.sm.frontier); // [Q] first tile that may have room
    // the group list: shared memory, or global memory when the mandatory arrays do not fit with it (read by this CTA only)
    const bool glist_sm = a.sm.glist != SM_NONE;
    uint2* s_glist = glist_sm ? reinterpret_cast<uint2*>(smem + a.sm.glist) : reinterpret_cast<uint2*>(a.glist_glob);   // [L*Q] (group, count)
    u32* s_gcl = glist_sm ? reinterpret_cast<u32*>(smem + a.sm.gcl) : a.glist_glob + 2 * HQS_MAX_GROUPS;             // [L*Q] class | level << 16
    // narrow remainders (exact amount = fr * gscale + rem): shared memory when they fit, else global scratch
    u64* p_rem = NARROW ? (a.sm.rem != SM_NONE ? reinterpret_cast<u64*>(smem + a.sm.rem) : reinterpret_cast<u64*>(a.rem_scratch)) : nullptr;
    const Cls* classes = a.sm.classes != SM_NONE ? reinterpret_cast<const Cls*>(smem + a.sm.classes) : reinterpret_cast<const Cls*>(a.classes);
    const uint8_t* vorder = a.sm.vorder != SM_NONE ? smem + a.sm.vorder : a.vorder;
    const uint8_t* blocked = a.blocked ? (a.sm.blocked != SM_NONE ? smem + a.sm.blocked : a.blocked) : nullptr;
    u32* s_bef = a.sm.bef != SM_NONE ? reinterpret_cast<u32*>(smem + a.sm.bef) : nullptr;
    u32* s_loc = a.sm.loc != SM_NONE ? reinterpret_cast<u32*>(smem + a.sm.loc) : nullptr;
    u32* s_kk = a.pf_shift ? (glist_sm ? reinterpret_cast<u32*>(smem + a.sm.kk) : a.glist_glob + 3 * HQS_MAX_GROUPS)
                           : nullptr;                                                  // [L*Q*2] tasks assigned per list entry (prefill)
    u32* s_top = a.pf_shift ? reinterpret_cast<u32*>(smem + a.sm.top) : nullptr;        // [Q] best level with waiting tasks left
    u32* s_pflvl = a.pf_shift ? reinterpret_cast<u32*>(smem + a.sm.pflvl) : nullptr;    // [Q] level of the class's prefilled tasks

    auto exact_of = [&](AT f, u32 w, int r) -> u64 {
        if constexpr (NARROW) return f == AMAX ? HQS_AMOUNT_MAX : (u64)f * a.gscale[r] + p_rem[(size_t)w * RT + r];
        else return f;
    };
    auto exact_amount = [&](const Var& dv, int r) -> u64 {
        if constexpr (NARROW) return (u64)dv.amount[r] * a.gscale[r];
        else return dv.amount[r];
    };
    // (re)stage the worker state from the tick input; thread per worker
    auto stage_workers = [&]() {
        for (u32 w = tid; w < W; w += blockDim.x) {
            u32 unt = 0;
#pragma unroll
            for (int r = 0; r < RT; ++r) {
                const u64 n = r < (int)R ? a.free_rw[(size_t)w * R + r] : 0;
                const u64 t = r < (int)R ? a.total_rw[(size_t)w * R + r] : 0;
                if constexpr (NARROW) {
                    const u64 g = a.gscale[r];
                    const u64 nq = g == 1 ? n : n / g;
                    s_fr[(size_t)w * RT + r] = n == HQS_AMOUNT_MAX ? AMAX : (AT)nq;
                    p_rem[(size_t)w * RT + r] = n == HQS_AMOUNT_MAX ? 0 : n - nq * g;
                } else {
                    s_fr[(size_t)w * RT + r] = n;
                }
                unt |= (t != 0 && n == t) ? (1u << r) : 0u;
                if (n != t) s_partial = 1;          // partly occupied at tick start: reservations are possible
            }
            s_unt[w] = unt;
            s_touch[w] = 0;
        }
    };
    // s_C[r] = sum over workers of the exact free amount, saturating (MAX absorbs); warp r handles resource r (+16 ...)
    auto sum_free_block = [&]() {
        for (u32 r = warp; r < R; r += TICK_WARPS) {
            u64 v = 0;
            for (u32 w = lane; w < W; w += 32) v = sat_add64(v, s_excl[w] ? 0 : exact_of(s_fr[(size_t)w * RT + r], w, (int)r));
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) v = sat_add64(v, __shfl_xor_sync(0xffffffffu, v, d));
            if (lane == 0) s_C[r] = v;
        }
    };

    // ---- prologue A: staging (overlaps the histogram of the worker CTAs)
    if (tid == 0) { s_nlist = 0; s_multi = 0; s_err = 0; s_final_err = 0; s_npacks = 0; s_partial = 0; s_npref = 0; s_bign = 0; s_xmis = 0; }
    if (tid < HQS_MAX_RESOURCES) { s_totmax[tid] = 0; s_D[tid] = 0; s_C[tid] = 0; }
    if (a.sm.classes != SM_NONE) {
        const uint4* src = reinterpret_cast<const uint4*>(a.classes);
        uint4* dst = reinterpret_cast<uint4*>(smem + a.sm.classes);
        for (u32 i = tid; i < a.classes_bytes / 16; i += blockDim.x) dst[i] = src[i];
    }
    if (a.sm.vorder != SM_NONE)
        for (u32 i = tid; i < Q * HQS_MAX_VARIANTS; i += blockDim.x) smem[a.sm.vorder + i] = a.vorder[i];
    if (a.blocked && a.sm.blocked != SM_NONE) {
        const u32 nb = W * Q;
        if ((nb & 15u) == 0 && ((size_t)a.blocked & 15u) == 0) {
            const uint4* src = reinterpret_cast<const uint4*>(a.blocked);
            uint4* dst = reinterpret_cast<uint4*>(smem + a.sm.blocked);
            for (u32 i = tid; i < nb / 16; i += blockDim.x) dst[i] = src[i];
        } else {
            for (u32 i = tid; i < nb; i += blockDim.x) smem[a.sm.blocked + i] = a.blocked[i];
        }
    }
    for (u32 w = tid; w < W; w += blockDim.x) {
        s_remtime[w] = a.rem_time[w];
        s_excl[w] = 0;
        if (a.min_util) a.excl_glob[w] = 0;
    }
    for (u32 c = tid; c < Q; c += blockDim.x) { s_front[c] = 0; s_noresv[c] = 0; }
    __syncthreads();
    stage_workers();
    // per-resource maximum of the (scaled) worker totals: a class no worker is big enough for is not demand
    for (u32 w = tid; w < W; w += blockDim.x) {
#pragma unroll
        for (int r = 0; r < RT; ++r) {
            if (r >= (int)R) continue;
            const u64 t = a.total_rw[(size_t)w * R + r];
            u64 tq = t;
            if constexpr (NARROW) tq = t == HQS_AMOUNT_MAX ? (u64)AMAX : (a.gscale[r] == 1 ? t : t / a.gscale[r]);
            atomicMax(reinterpret_cast<unsigned long long*>(&s_totmax[r]), (unsigned long long)tq);
        }
    }
    // groups without ready tasks keep k = 0 (the emit step's chunk filter reads k of every group)
    for (u32 g = tid; g < G; g += blockDim.x) { a.gout[g].k = 0; if (a.pf_shift) a.gout2[g] = make_uint4(0, 0, 0, 0); }
    __syncthreads();
    sum_free_block();

    // ---- prologue B: wait for the histogram; sharded: exchange the count vectors over NVLink
    if (a.flags & TF_COUNT) {
        if (tid == 0 && !spin_until_ge(&a.sync->count_done, nW)) s_err = 21;        // the histogram never completed
    }
    __syncthreads();
    const long long t_counted = clock64();
    const u32* tot_all = a.total_ext ? a.total_ext : a.total_local;
    const u32* before = a.before_ext;
    if (a.x_world) {
        // block-strided peer stores of my count vector into every rank's exchange buffer (own included), a system
        // fence, then one release flag per peer; afterwards acquire every rank's flag of THIS tick.  Next to the flags every
        // rank publishes its group count G: a rank with another G (e.g. proactive filling on one rank only) lays its vector
        // out differently, and summing it would solve on garbage, so the tick fails before anything is emitted.  Only G is
        // compared; ranks with equal G but another prefill reserve / max or level / class set are not detected.
        const u32 parity = a.x_seq & 1u;
        for (u32 r = 0; r < a.x_world; ++r) {
            u32* dst = a.x_peer[r] + ((size_t)parity * HQS_MAX_PEERS + a.x_rank) * HQS_MAX_GROUPS;
            for (u32 g = tid; g < G; g += blockDim.x) dst[g] = __ldcg(a.total_local + g);
            if (tid == 0) a.x_peer[r][(size_t)2 * HQS_MAX_PEERS * HQS_MAX_GROUPS + (2 + parity) * HQS_MAX_PEERS + a.x_rank] = G;
        }
        __threadfence_system();
        __syncthreads();
        if (tid < a.x_world) {
            u32* flags = a.x_peer[tid] + (size_t)2 * HQS_MAX_PEERS * HQS_MAX_GROUPS + (size_t)parity * HQS_MAX_PEERS;
            st_release_sys(flags + a.x_rank, a.x_seq);
        }
        if (tid < a.x_world) {
            const u32* myflags = a.x_peer[a.x_rank] + (size_t)2 * HQS_MAX_PEERS * HQS_MAX_GROUPS + (size_t)parity * HQS_MAX_PEERS;
            const long long t0 = clock64();
            bool got = true;
            while (ld_acquire_sys(myflags + tid) != a.x_seq) {
                if (clock64() - t0 > PEER_TIMEOUT_CYCLES) { s_err = 22 + (tid << 8); got = false; break; }       // peer `tid` never sent its counts
                __nanosleep(32);
            }
            const u32 pg = got ? __ldcg(myflags + 2 * HQS_MAX_PEERS + tid) : G;          // the peer's G (after its flag)
            if (pg != G) atomicCAS(&s_xmis, 0u, 0x80000000u | (tid << 16) | pg);
        }
        __syncthreads();
        // on a mismatch the solve runs on an empty ready set and the tick ends with error 4
        const bool xmis = s_xmis != 0;
        const u32* xc = a.x_peer[a.x_rank] + (size_t)parity * HQS_MAX_PEERS * HQS_MAX_GROUPS;
        for (u32 g = tid; g < G; g += blockDim.x) {
            u32 all = 0, bef = 0;
            for (u32 r = 0; r < a.x_world; ++r) {
                const u32 v = __ldcg(xc + (size_t)r * HQS_MAX_GROUPS + g);     // peers wrote it: bypass L1
                all += v;
                bef += r < a.x_rank ? v : 0u;
            }
            a.x_all[g] = xmis ? 0u : all;
            a.x_before[g] = xmis ? 0u : bef;
        }
        __syncthreads();
        tot_all = a.x_all;
        before = a.x_before;
    }

    // ---- prologue C: compact the non-empty groups in processing order: level asc (= priority desc), then the
    //      tick's class order.  Every warp owns a contiguous range of positions; two passes, one barrier.
    {
        const u32 n_pos = (a.L * Q) << a.pf_shift;
        const u32 seg = ((n_pos + TICK_WARPS - 1) / TICK_WARPS + 31) & ~31u;      // positions per warp, multiple of 32
        u32 nn[HQS_MAX_GROUPS / TICK_WARPS / 32], gg[HQS_MAX_GROUPS / TICK_WARPS / 32];
        u32 cnt = 0;
#pragma unroll
        for (int i = 0; i < (int)(HQS_MAX_GROUPS / TICK_WARPS / 32); ++i) {
            nn[i] = 0; gg[i] = 0;
            const u32 pos = warp * seg + i * 32 + lane;
            if ((u32)i * 32 < seg && pos < n_pos) {
                const u32 pos2 = pos >> a.pf_shift;                   // (level, class position); the low bit of pos: prefilled sub-group
                const u32 lvl = pos2 / Q, j = pos2 - lvl * Q;
                gg[i] = ((lvl * Q + a.order[j]) << a.pf_shift) | (pos & a.pf_shift);
                nn[i] = __ldcg(tot_all + gg[i]);
            }
            cnt += __popc(__ballot_sync(0xffffffffu, nn[i] != 0));
        }
        if (lane == 0) s_wcnt[warp] = cnt;
        __syncthreads();
        u32 off = 0, tot = 0;
        for (u32 w2 = 0; w2 < TICK_WARPS; ++w2) { const u32 c2 = s_wcnt[w2]; off += w2 < warp ? c2 : 0; tot += c2; }
#pragma unroll
        for (int i = 0; i < (int)(HQS_MAX_GROUPS / TICK_WARPS / 32); ++i) {
            const u32 bal = __ballot_sync(0xffffffffu, nn[i] != 0);
            if (nn[i]) {
                const u32 slot = off + __popc(bal & ((1u << lane) - 1));
                const u32 g = gg[i];
                s_glist[slot] = make_uint2(g, nn[i]);
                s_gcl[slot] = ((g >> a.pf_shift) % Q) | (((g >> a.pf_shift) / Q) << 16);
                if (before) {
                    if (s_bef) { s_bef[slot] = __ldcg(before + g); s_loc[slot] = __ldcg(a.total_local + g); }
                }
            }
            off += __popc(bal);
        }
        if (tid == 0) s_nlist = tot;
        __syncthreads();
    }
    const u32 n_list = s_nlist;
    // ---- prologue D: can ANY level be saturated?  If every class has one variant and no `All` entry, a level's
    //      demand never exceeds (total demand - what earlier levels consumed), so "total demand fits the pool"
    //      rules saturation out for the whole tick and the per-level tests are skipped (mode M1).
    bool skip_sat = (a.flags & TF_PACK) == 0;
    {
        u64 val[RT];
#pragma unroll
        for (int r = 0; r < RT; ++r) val[r] = 0;
        u32 multi = 0;
        for (u32 e = tid; e < n_list; e += blockDim.x) {
            const u32 c = s_gcl[e] & 0xFFFFu, n = s_glist[e].y;
            const Cls& cl = classes[c];
            if (cl.n_variants > 1) multi = 1;
            if (n > WIDE_MAX_GROUP) s_bign = 1;
            const Var& dv = cl.v[vorder[c * HQS_MAX_VARIANTS]];
            if (dv.all_mask) multi = 1;
            bool servable = true;
#pragma unroll
            for (int r = 0; r < RT; ++r) servable &= (u64)dv.amount[r] <= s_totmax[r];
            if (servable) {
#pragma unroll
                for (int r = 0; r < RT; ++r) val[r] = sat_add64(val[r], sat_mul64(exact_amount(dv, r), (u64)n));
            }
        }
#pragma unroll
        for (int r = 0; r < RT; ++r) {
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) val[r] = sat_add64(val[r], __shfl_xor_sync(0xffffffffu, val[r], d));
        }
        if (__any_sync(0xffffffffu, multi) && lane == 0) s_multi = 1;
        if (lane == 0) {
#pragma unroll
            for (int r = 0; r < RT; ++r) s_red[warp * RT + r] = val[r];
        }
        __syncthreads();
        if (tid < RT) {
            u64 d = 0;
            for (u32 w2 = 0; w2 < TICK_WARPS; ++w2) d = sat_add64(d, s_red[w2 * RT + tid]);
            s_D[tid] = d;
        }
        __syncthreads();
        bool fits = s_multi == 0;
        for (u32 r = 0; r < R; ++r) fits &= s_C[r] == HQS_AMOUNT_MAX || s_D[r] <= s_C[r];
        skip_sat = skip_sat || fits;
    }
    // plain tick: one variant per class, no `All`, no blocked mask, no time limits, no minimum utilisation.  Its
    // first-fit runs in the lean loop below (worker tile in registers, next group prefetched).
    const bool plain = s_multi == 0 && !blocked && !a.any_time_limit && !a.min_util;
    __syncthreads();
    const long long t_prologue = clock64();

    // =============================================================================================
    // wide lean first-fit (plain ticks without reservations / proactive filling, pools of up to 512 workers): EVERY worker
    // is a lane.  Warp j holds the free vectors of workers 32 j .. 32 j + 31 in registers for the whole loop, so a group
    // costs ONE step for the whole pool instead of one step per visited tile of a single warp: fit count per lane, warp
    // sum, exchange of the warp sums through shared memory (one 8-byte record per warp and group, double-buffered, one
    // named barrier), prefix over the warps, and only the warps the group reaches scan their lanes and take.  The result
    // is exactly the first-fit of the one-warp loop (ascending worker id); the class frontiers are not needed.  Count
    // segments: a warp with takers knows that every warp below it is a full taker, so its segment index is the running
    // base + the non-zero lanes below it; the number of segments a warp wrote travels in its record of the NEXT group,
    // so the group record of warp 0 trails by one group.  A class nobody could take a task of is dead for the rest of
    // the loop (free amounts only shrink here): its later groups are skipped without an exchange.
    // =============================================================================================
    struct WideOut { u32 seg_base, out_base, steps; bool overflow; };
    constexpr int WIDE_WORDS = RT * (int)(sizeof(AT) / 4);                      // registers of one free vector
    const bool wide_ok = plain && !s_bign && !(a.flags & TF_NO_WIDE) && WIDE_WORDS <= 16 && n_tiles <= TICK_WARPS && a.sm.classes != SM_NONE;
    auto run_wide = [&]() -> WideOut {
        const u32 li0 = s_blk[1];
        u32 out_base = s_blk[2], seg_cur = s_blk[3];
        const u32 nw = n_tiles;                        // participating warps: one tile of 32 workers each
        WideOut res;
        res.seg_base = seg_cur; res.out_base = out_base; res.steps = 0; res.overflow = false;
        uint8_t* s_dead = s_noresv;                    // [Q], all zero here (reservations are off in this loop)
        // the class table through a pointer the compiler knows to be shared memory (`classes` is shared-or-global: generic loads)
        const Cls* cls_s = reinterpret_cast<const Cls*>(smem + a.sm.classes);
        if (warp < nw) {
            const u32 lt_mask = (1u << lane) - 1;
            const u32 wk = warp * 32 + lane;
            const bool in_pool = wk < W;
            AT fr[RT];
#pragma unroll
            for (int r = 0; r < RT; ++r) fr[r] = in_pool ? s_fr[(size_t)wk * RT + r] : 0;
            u32 par = 0, cme_prev = 0;
            bool pend = false;
#ifdef HQS_TRACE
            u32 tw[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#define TWC() ([] { u32 c_; asm volatile("mov.u32 %0, %%clock;" : "=r"(c_)::"memory"); return c_; }())
            u32 tw_prev = TWC();
#define TW(i) { const u32 c__ = TWC(); tw[i] += c__ - tw_prev; tw_prev = c__; }
#else
#define TW(i)
#endif
            u32 p_g = 0, p_k = 0, p_out = 0, p_seglo = 0;      // warp 0: the record that waits for its segment count
            uint2 ge_n = s_glist[li0];
            u32 c_n = s_gcl[li0] & 0xFFFFu;
            Var dv_n = cls_s[c_n].v[0];
            u32 dead_n = s_dead[c_n];
            for (u32 e = li0; e < n_list; ++e) {
                const uint2 ge = ge_n;
                const u32 c = c_n;
                Var dv = dv_n;
                dv.all_mask = 0;                                   // plain tick: lets the compiler drop the `All` arm
                const u32 dead = dead_n;
                if (e + 1 < n_list) {
                    ge_n = s_glist[e + 1];
                    c_n = s_gcl[e + 1] & 0xFFFFu;
                    dv_n = cls_s[c_n].v[0];
                    dead_n = s_dead[c_n];
                }
                if (dead) continue;                                // k stays 0 (prologue)
                const u32 g = ge.x, n = ge.y;
                par ^= 1u;
                TW(0)                                              // loop top: entry, prefetch of the next group
                // ---- fit count of my lane, warp sum (clamped to n: prefixes stay below 2^32), record out
                const u32 cnt = in_pool ? (u32)fit_count<RT>(fr, 0u, dv, (u64)n) : 0u;
                TW(1)                                              // fit count
                u32 total = __reduce_add_sync(0xffffffffu, cnt);
                total = total < n ? total : n;
                const u32 nzm = __ballot_sync(0xffffffffu, cnt != 0);
                if (lane == 0)       // one 8-byte record: total (27 bits) | non-zero lanes (6) << 27 | my segments of the previous group << 34
                    s_wx[par][warp] = (unsigned long long)total | ((unsigned long long)__popc(nzm) << 27) | ((unsigned long long)cme_prev << 34);
                TW(2)                                              // warp sum, vote, record
                // ---- the other warps' records of this group (double-buffered: one barrier per group is enough)
                bar_named(3, nw * 32);
                u32 tj = 0, nzj = 0, cprev = 0;
                if (lane < nw) {
                    const unsigned long long v = s_wx[par][lane];
                    tj = (u32)v & 0x07FFFFFFu; nzj = (u32)(v >> 27) & 0x7Fu; cprev = (u32)(v >> 34) & 0x7Fu;
                }
                TW(3)                                              // exchange
                const u32 base = __reduce_add_sync(0xffffffffu, lane < warp ? tj : 0u);
                const u32 all = __reduce_add_sync(0xffffffffu, tj);
                const u32 nzb = __reduce_add_sync(0xffffffffu, lane < warp ? nzj : 0u);
                const u32 sprev = __reduce_add_sync(0xffffffffu, cprev);
                // the previous group's segments are counted now: its record (warp 0), my segment base
                if (warp == 0 && lane == 0 && pend) {
                    GroupOut go;
                    go.k = p_k; go.out_off = p_out; go.seg_lo = p_seglo; go.seg_n = sprev;
                    a.gout[p_g] = go;
                }
                seg_cur += sprev;
                if (seg_cur > SEG_CAP) { res.overflow = true; seg_cur = SEG_CAP; }
                TW(4)                                              // prefix over the warps, previous record
                // ---- take: lanes in worker order until n is handed out.  Only a warp that the group reaches scans its lanes.
                u32 cme = 0;
                if (base < n && nzm != 0) {
                    const u32 room = n - base;                     // what the warps below me left
                    u32 inc = cnt;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const u32 y = __shfl_up_sync(0xffffffffu, inc, d);
                        if ((int)lane >= d) inc += y;
                    }
                    const u32 exl = inc - cnt;
                    TW(5)                                          // scan
                    u32 take = 0;
                    if (cnt && exl < room) take = min(cnt, room - exl);
                    const u32 tkm = __ballot_sync(0xffffffffu, take != 0);
                    if (take) {
                        const u32 si = seg_cur + nzb + __popc(tkm & lt_mask);
                        if (si < SEG_CAP) { a.seg_cum[si] = base + exl + take; a.seg_wv[si] = wk; }
                    }
                    // an unused resource has amount 0 (hqs_classes_set), `All` does not occur in a plain tick: branch-free
#pragma unroll
                    for (int r = 0; r < RT; ++r) fr[r] = fr[r] == AMAX ? fr[r] : fr[r] - (AT)take * dv.amount[r];
                    cme = __popc(tkm);
                }
                cme_prev = cme;
                TW(6)                                              // takes, segments
                const u32 k = all < n ? all : n;
                if (all == 0) {                                    // nobody can take a task of the class any more
                    if (lane == 0) s_dead[c] = 1;
                    if (c_n == c) dead_n = 1;
                    __syncwarp();
                }
                if (warp == 0) {
                    u32 k_loc = k;
                    if (before) {
                        const u32 bef = s_bef ? s_bef[e] : __ldcg(before + g);
                        const u32 loc = s_loc ? s_loc[e] : __ldcg(a.total_local + g);
                        k_loc = k > bef ? k - bef : 0;
                        k_loc = k_loc < loc ? k_loc : loc;
                    }
                    p_g = g; p_k = k; p_out = out_base; p_seglo = seg_cur; pend = true;
                    out_base += k_loc;
                    ++res.steps;
                }
                TW(7)                                              // group record
            }
#ifdef HQS_TRACE
            if (warp == 0 && lane == 0)
                for (int q = 0; q < 8; ++q) s_trw[q] = tw[q];
#endif
            // free vectors back to shared memory
            if (in_pool) {
#pragma unroll
                for (int r = 0; r < RT; ++r) s_fr[(size_t)wk * RT + r] = fr[r];
            }
            if (lane == 0) s_wc[warp] = cme_prev;
            bar_named(2, TICK_THREADS);
            if (warp == 0) {
                // the last group's segment count
                const u32 clast = lane < nw ? s_wc[lane] : 0u;
                const u32 slast = __reduce_add_sync(0xffffffffu, clast);
                if (lane == 0 && pend) {
                    GroupOut go;
                    go.k = p_k; go.out_off = p_out; go.seg_lo = p_seglo; go.seg_n = slast;
                    a.gout[p_g] = go;
                }
                seg_cur += slast;
                if (seg_cur > SEG_CAP) { res.overflow = true; seg_cur = SEG_CAP; }
                res.seg_base = seg_cur; res.out_base = out_base;
            }
        } else {
            bar_named(2, TICK_THREADS);
        }
        return res;
    };
#undef TW
#ifdef HQS_TRACE
#undef TWC
#endif

    // =============================================================================================
    // block-parallel steps, executed by ALL warps of the CTA (the solver warp calls block_work after waking the others)
    // =============================================================================================
    auto block_work = [&](u32 cmd) {
        if (cmd == BLK_WIDE) { run_wide(); return; }
        if (cmd == BLK_RESTART) {
            // min-utilisation restart: excluded workers stay out, everything else starts over
            stage_workers();
            for (u32 c = tid; c < Q; c += blockDim.x) { s_front[c] = 0; s_noresv[c] = 0; }
            for (u32 w = tid; w < W; w += blockDim.x)
                if (s_excl[w] == 2) s_excl[w] = 0;         // reservations are made again by the new pass
            bar_named(2, TICK_THREADS);
            return;
        }
        if (cmd == BLK_PREFILL) {
            // ---- proactive filling (mapping.rs:156-230; specification: tests/greedy_model.py::_with_prefill).  For every
            //      class whose best level with waiting (not prefilled) tasks left is the best one over all classes:
            //      size = waiting tasks left at that level - reserve (0 while the class holds prefilled tasks at another
            //      level); eligible workers = those that got an assignment of the class in this tick and hold no prefilled
            //      task of it; each gets min(size / eligible, max) of the next waiting tasks.  Result: a prefill range behind
            //      the assigned ranks of the (level, class) group, as segments of its own (gout2, pf_cum, pf_wk).
            const u32 pfs = a.pf_shift;
            for (u32 c = tid; c < Q; c += blockDim.x) { s_top[c] = 0xFFFFFFFFu; s_pflvl[c] = 0xFFFFFFFFu; }
            if (tid == 0) { s_blk[6] = 0xFFFFFFFFu; s_blk[7] = 0; s_qT[0] = 0; s_qT[1] = 0; }
            bar_named(2, TICK_THREADS);
            for (u32 e = tid; e < n_list; e += blockDim.x) {
                const u32 c = s_gcl[e] & 0xFFFFu, lvl = s_gcl[e] >> 16;
                const u32 left = s_glist[e].y - s_kk[e];
                if (left) atomicMin((s_glist[e].x & pfs) ? &s_pflvl[c] : &s_top[c], lvl);
            }
            bar_named(2, TICK_THREADS);
            u32 best = 0xFFFFFFFFu;
            for (u32 c = tid; c < Q; c += blockDim.x) best = min(best, s_top[c]);
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, d));
            if (lane == 0 && best != 0xFFFFFFFFu) atomicMin(&s_blk[6], best);
            bar_named(2, TICK_THREADS);
            const u32 gtop = s_blk[6];
            u32 pf_out = 0, pf_seg = 0;                                          // uniform running totals
            if (gtop != 0xFFFFFFFFu) {
                for (u32 c = 0; c < Q; ++c) {
                    if (s_top[c] != gtop || (s_pflvl[c] != 0xFFFFFFFFu && s_pflvl[c] != gtop)) continue;      // uniform
                    // the (gtop, c, waiting) entry
                    bar_named(2, TICK_THREADS);                                  // the previous candidate's readers are done
                    if (tid == 0) s_blk[7] = 0xFFFFFFFFu;
                    for (u32 w = tid; w < W; w += blockDim.x) s_touch[w] = 0;     // reused: worker got an assignment of the class
                    bar_named(2, TICK_THREADS);
                    for (u32 e = tid; e < n_list; e += blockDim.x) {
                        if ((s_gcl[e] & 0xFFFFu) != c || (s_glist[e].x & pfs)) continue;
                        if ((s_gcl[e] >> 16) == gtop) s_blk[7] = e;
                        if (s_kk[e]) {
                            const uint4 go = *reinterpret_cast<const uint4*>(a.gout + s_glist[e].x);        // written by this CTA
                            for (u32 q = 0; q < go.w; ++q) s_touch[a.seg_wv[go.z + q] & 0xFFFFu] = 1;
                        }
                    }
                    bar_named(2, TICK_THREADS);
                    const u32 et = s_blk[7];
                    const u32 k = s_kk[et], left = s_glist[et].y - k;
                    if (left <= a.pf_reserve) continue;                          // uniform
                    const u32 size = left - a.pf_reserve;
                    // eligible workers in ascending order (warp 0 compacts tile by tile into s_td, free at this point)
                    if (warp == 0) {
                        u32 n_el = 0;
                        for (u32 tile = 0; tile < n_tiles; ++tile) {
                            const u32 w = tile * 32 + lane;
                            const bool el = w < W && s_touch[w] && !(a.prefilled_wc && a.prefilled_wc[(size_t)w * Q + c]);
                            const u32 em = __ballot_sync(0xffffffffu, el);
                            if (el) s_td[n_el + __popc(em & ((1u << lane) - 1))] = (unsigned short)w;
                            n_el += __popc(em);
                        }
                        if (lane == 0) s_qT[2] = n_el;
                    }
                    bar_named(2, TICK_THREADS);
                    const u32 n_el = (u32)s_qT[2];
                    if (n_el == 0) continue;                                     // uniform
                    const u32 ps = min(size / n_el, a.pf_max);
                    if (ps == 0 || pf_seg + n_el > PF_SEG_CAP) continue;         // uniform
                    for (u32 i = tid; i < n_el; i += blockDim.x) {
                        a.pf_cum[pf_seg + i] = k + (i + 1) * ps;
                        a.pf_wk[pf_seg + i] = s_td[i];
                    }
                    if (tid == 0) a.gout2[s_glist[et].x] = make_uint4(k + n_el * ps, pf_out, pf_seg, n_el);
                    // records of this rank: a sharded tick emits only the part of the range [k, k + n_el * ps) that falls
                    // into its own ranks [bef, bef + loc) of the group, so the offsets behind the assignments are local
                    // (the sharded inputs are re-derived from `a` here rather than captured from the solve's scope, which
                    // would keep them live in registers through the plain tick's solve)
                    u32 share = n_el * ps;
                    const u32* bef_g = a.x_world ? a.x_before : a.before_ext;
                    if (bef_g) {
                        const u32 g = s_glist[et].x;
                        const bool sm = a.sm.bef != SM_NONE;
                        const u32 bef = sm ? reinterpret_cast<const u32*>(smem + a.sm.bef)[et] : __ldcg(bef_g + g);
                        const u32 loc = sm ? reinterpret_cast<const u32*>(smem + a.sm.loc)[et] : __ldcg(a.total_local + g);
                        const u32 lo = max(k, bef), hi = min(k + n_el * ps, bef + loc);
                        share = hi > lo ? hi - lo : 0u;
                    }
                    pf_out += share;
                    pf_seg += n_el;
                    bar_named(2, TICK_THREADS);
                }
            }
            if (tid == 0) s_blk[7] = pf_out;
            __threadfence();
            bar_named(2, TICK_THREADS);
            return;
        }
        // ---- BLK_PACK: the level [li, lj) is saturated
        const u32 li = s_blk[1], lj = s_blk[2], region0 = s_blk[3];
        const u32 ng = lj - li;
        const double phi = __hiloint2double((int)s_blk[5], (int)s_blk[4]);
        if (tid < PACK_MAX_CAND) s_qT[tid] = 0;
        if (tid == 0) {
            u32 ci = 0;
            for (u32 e = li; e < lj; ++e) {
                const u32 c = s_gcl[e] & 0xFFFFu;
                s_cbase[e - li] = ci;
                for (u32 v = 0; v < classes[c].n_variants; ++v) a.pk.cand[ci++] = c | (v << 16) | ((e - li) << 24);
            }
            s_cbase[ng] = ci;
            a.pk.meta[0] = ci;
            a.pk.meta[1] = ng;
        }
        bar_named(2, TICK_THREADS);
        // a. quotas: share of each class proportional to how many fit on the worker alone.  Pass 1: every worker's
        //    own count per group (stashed in its quota slot) and the pool sums; pass 2: the quotas.
        for (u32 w0 = 0; w0 < W; w0 += blockDim.x) {
            const u32 w = w0 + tid;
            const bool has = w < W && !s_excl[w];
            AT fr[RT];
#pragma unroll
            for (int r = 0; r < RT; ++r) fr[r] = has ? s_fr[(size_t)w * RT + r] : 0;
            const u32 unt = has ? s_unt[w] : 0;
            const u64 rt = has ? s_remtime[w] : 0;
            for (u32 e = li; e < lj; ++e) {
                const u32 c = s_gcl[e] & 0xFFFFu, n = s_glist[e].y;
                u64 cn = 0;
                if (has) {
                    const uint8_t blk = blocked ? blocked[(size_t)w * Q + c] : 0;
                    for (u32 v = 0; v < classes[c].n_variants; ++v) {
                        const Var& dv = classes[c].v[v];
                        if (!admissible(dv, v, blk, rt)) continue;
                        const u64 f = fit_count<RT>(fr, unt, dv, n);
                        cn = f > cn ? f : cn;
                    }
                }
                if (w < W) a.pk.quota[(size_t)w * PACK_MAX_CAND + (e - li)] = (u32)cn;       // cn <= n < 2^32
                u64 x = cn;
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d);
                if (lane == 0 && x) atomicAdd(reinterpret_cast<unsigned long long*>(&s_qT[e - li]), (unsigned long long)x);
            }
        }
        bar_named(2, TICK_THREADS);
        for (u32 w = tid; w < W; w += blockDim.x) {
            for (u32 e = li; e < lj; ++e) {
                const u32 n = s_glist[e].y;
                const u64 T = s_qT[e - li];
                const u64 cn = a.pk.quota[(size_t)w * PACK_MAX_CAND + (e - li)];           // this thread's own store
                const u64 q = T ? ((u64)n * cn + T - 1) / T : 0;
                const u64 q_phi = __double2ull_ru(__dmul_rn(__ull2double_rn(q), phi));     // ceil(q * phi)
                a.pk.quota[(size_t)w * PACK_MAX_CAND + (e - li)] = (u32)q_phi;
            }
            // b. publish the worker state for the pack warps
#pragma unroll
            for (int r = 0; r < RT; ++r)
                if (r < (int)R) a.pk.fr[(size_t)w * R + r] = exact_of(s_fr[(size_t)w * RT + r], w, r);
            if (a.min_util) a.excl_glob[w] = s_excl[w];
        }
        __threadfence();
        bar_named(2, TICK_THREADS);
        if (tid == 0) {
            const u32 np = s_npacks + 1;
            s_npacks = np;
            st_release(&a.sync->cmd, (np << 2) | CMD_PACK);
            if (!spin_until_ge(&a.sync->pack_done, np * nW)) s_err = 23;
        }
        bar_named(2, TICK_THREADS);
        // c. the workers filled themselves: take their free vectors back
        for (u32 w = tid; w < W; w += blockDim.x) {
#pragma unroll
            for (int r = 0; r < RT; ++r)
                if (r < (int)R) {
                    const u64 x = __ldcg(a.pk.fr + (size_t)w * R + r);
                    if constexpr (NARROW) {
                        const u64 g = a.gscale[r], rm = p_rem[(size_t)w * RT + r];
                        s_fr[(size_t)w * RT + r] = x == HQS_AMOUNT_MAX ? AMAX : (AT)(g == 1 ? x - rm : (x - rm) / g);
                    } else {
                        s_fr[(size_t)w * RT + r] = x;
                    }
                }
        }
        bar_named(2, TICK_THREADS);
        // d. cap what the workers took for each class at its count, (variant, worker) order: one warp per group of the
        //    level, count segments into the group's own region.  The excess (what a worker took beyond the class count)
        //    replaces the worker's `taken` entry; the solver warp hands it back when it reaches the group — the
        //    specification interleaves hand-backs and first-fit group by group.
        for (u32 gi = warp; gi < ng; gi += TICK_WARPS) {
            const u32 e = li + gi;
            const u32 c = s_gcl[e] & 0xFFFFu, n = s_glist[e].y;
            const u32 nv = classes[c].n_variants;
            const u32 seglo = region0 + 2u * W * s_cbase[gi];
            u32 pos = 0, nseg = 0, ex_lo = 0xFFFFu, ex_hi = 0;
            for (u32 v = 0; v < nv; ++v) {
                const Var& dv = classes[c].v[v];
                for (u32 tile = 0; tile < n_tiles; ++tile) {
                    const u32 w = tile * 32 + lane;
                    u32* tk = a.pk.taken + (size_t)w * PACK_MAX_CAND + s_cbase[gi] + v;
                    const u32 k = w < W ? __ldcg(tk) : 0;
                    if (__ballot_sync(0xffffffffu, k != 0) == 0) continue;
                    u64 inc = k;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const u64 y = __shfl_up_sync(0xffffffffu, inc, d);
                        if ((int)lane >= d) inc += y;
                    }
                    const u64 room = n - pos, exc = inc - k;
                    u32 use = 0;
                    if (k && exc < room) use = (u32)((u64)k < room - exc ? (u64)k : room - exc);
                    const u32 um = __ballot_sync(0xffffffffu, use != 0);
                    if (use) {
                        const u32 si = seglo + nseg + __popc(um & ((1u << lane) - 1));
                        if (si < SEG_CAP) { a.seg_cum[si] = pos + (u32)exc + use; a.seg_wv[si] = w | (v << 16); }
                        // what stays on the worker makes its resources "touched" (free != total); an unbounded amount stays
                        u32 touched = 0;
#pragma unroll
                        for (int r = 0; r < RT; ++r)
                            if (((dv.used_mask >> r) & 1) && s_fr[(size_t)w * RT + r] != AMAX) touched |= 1u << r;
                        atomicAnd(&s_unt[w], ~touched);
                        s_touch[w] = 1;
                    }
                    if (k) *tk = k - use;
                    if (__ballot_sync(0xffffffffu, k > use)) { ex_lo = ex_lo < tile ? ex_lo : tile; ex_hi = ex_hi > tile + 1 ? ex_hi : tile + 1; }
                    nseg += __popc(um);
                    const u64 total = __shfl_sync(0xffffffffu, inc, 31);
                    pos += (u32)(total < room ? total : room);
                }
            }
            if (lane == 0) { s_pkpos[gi] = pos; s_pknseg[gi] = nseg; s_pkseglo[gi] = seglo; s_pkex[gi] = ex_lo | (ex_hi << 16); }
        }
        __threadfence();
        bar_named(2, TICK_THREADS);
        // e. frontiers of the level's single-variant classes on what the pack left: the first worker that can still take
        //    one task (one warp per group; the solver warp alone would find out tile by tile, group by group).  Hand-backs
        //    lower the frontiers again where free amounts grow.
        if (!(a.flags & TF_NO_REFRESH)) {
            for (u32 gi = warp; gi < ng; gi += TICK_WARPS) {
                const u32 c = s_gcl[li + gi] & 0xFFFFu;
                if (classes[c].n_variants != 1) continue;
                const Var& dv = classes[c].v[0];
                const u32 old = s_front[c];
                u32 res = n_tiles * 32;
                for (u32 tile = old >> 5; tile < n_tiles; ++tile) {
                    const u32 w = tile * 32 + lane;
                    u64 cnt = 0;
                    if (w < W && !s_excl[w]) {
                        AT fr[RT];
#pragma unroll
                        for (int r = 0; r < RT; ++r) fr[r] = s_fr[(size_t)w * RT + r];
                        const uint8_t blk = blocked ? blocked[(size_t)w * Q + c] : 0;
                        const u64 rt = a.any_time_limit ? s_remtime[w] : HQS_TIME_INF;
                        if (admissible(dv, 0, blk, rt)) cnt = fit_count<RT>(fr, s_unt[w], dv, 1);
                    }
                    const u32 m = __ballot_sync(0xffffffffu, cnt != 0);
                    if (m) { res = tile * 32 + (u32)__ffs(m) - 1; break; }
                }
                if (lane == 0 && res > old) s_front[c] = (unsigned short)res;
            }
            bar_named(2, TICK_THREADS);
        }
    };

    // ---- reservations (solver.rs:133-151; specification: tests/greedy_model.py::_Tick.reserve).  A class that is left
    //      with unplaced tasks claims workers that are big enough for it by their TOTALS but cannot take one task of it at
    //      tick start: such a worker receives nothing in this tick.  Only workers without any assignment in this tick, at
    //      most one per unplaced task, highest worker index first, and only while the class's count does not exceed the
    //      batch limit (every capable worker counts at least once, batches.rs:80-91).  Rare path: exact 64-bit arithmetic
    //      on the tick input.
    const ClassT<RT, u64>* classes64 = reinterpret_cast<const ClassT<RT, u64>*>(a.classes64);
    auto reserve_for = [&](u32 c, u32 n_all, u32 remaining) {
        const ClassT<RT, u64>& cl = classes64[c];
        const u32 nv = cl.n_variants;
        u64 limit = 0;
        // per lane and tile: capable by totals?  how many fit at tick start (sum over variants, 1024 each)?
        for (u32 tile = 0; tile < n_tiles; ++tile) {
            const u32 w = tile * 32 + lane;
            u64 lim_w = 0;
            if (w < W) {
                const u64 rt = s_remtime[w];
                bool cap = false;
                u64 fits = 0;
                for (u32 v = 0; v < nv; ++v) {
                    const VarT<RT, u64>& dv = cl.v[v];
                    bool ok = rt == HQS_TIME_INF || dv.min_time_ms <= rt;
                    u64 cnt = HQS_AMOUNT_MAX;
#pragma unroll
                    for (int r = 0; r < RT; ++r) {
                        if (r >= (int)R || !((dv.used_mask >> r) & 1)) continue;
                        const u64 t = a.total_rw[(size_t)w * R + r], f = a.free_rw[(size_t)w * R + r];
                        if ((dv.all_mask >> r) & 1) { ok &= t != 0; cnt = cnt < (f != 0 ? 1ull : 0ull) ? cnt : (f != 0 ? 1ull : 0ull); }
                        else { ok &= dv.amount[r] <= t; if (f != HQS_AMOUNT_MAX) { const u64 q = f / dv.amount[r]; cnt = cnt < q ? cnt : q; } }
                    }
                    cap |= ok;
                    fits += cnt < 1024 ? cnt : 1024;
                }
                if (cap) lim_w = fits > 1 ? fits : 1;
            }
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) lim_w += __shfl_xor_sync(0xffffffffu, lim_w, d);
            limit += lim_w;
        }
        u32 got = 0;
        if ((u64)n_all <= limit) {
            for (u32 tile = n_tiles; tile-- > 0 && got < remaining;) {
                const u32 w = tile * 32 + lane;
                bool elig = false;
                if (w < W && !s_excl[w] && !s_touch[w]) {
                    const u64 rt = s_remtime[w];
                    bool cap = false, fits_now = false;
                    for (u32 v = 0; v < nv; ++v) {
                        const VarT<RT, u64>& dv = cl.v[v];
                        bool ok = rt == HQS_TIME_INF || dv.min_time_ms <= rt;
                        bool one = true;
#pragma unroll
                        for (int r = 0; r < RT; ++r) {
                            if (r >= (int)R || !((dv.used_mask >> r) & 1)) continue;
                            const u64 t = a.total_rw[(size_t)w * R + r], f = a.free_rw[(size_t)w * R + r];
                            if ((dv.all_mask >> r) & 1) { ok &= t != 0; one &= f != 0; }
                            else { ok &= dv.amount[r] <= t; one &= f == HQS_AMOUNT_MAX || dv.amount[r] <= f; }
                        }
                        cap |= ok;
                        fits_now |= one;
                    }
                    elig = cap && !fits_now;
                }
                const u32 em = __ballot_sync(0xffffffffu, elig);
                // the highest (remaining - got) eligible lanes of the tile
                const u32 above = __popc(em & ~((2u << lane) - 1u));          // eligible lanes with a higher index
                if (elig && above < remaining - got) s_excl[w] = 2;
                got += min((u32)__popc(em), remaining - got);
            }
        }
        if (got < remaining && lane == 0) s_noresv[c] = 1;    // eligibility only shrinks during a tick
        __syncwarp();
    };

    // =============================================================================================
    // the solver warp
    // =============================================================================================
    u32 n_assigned = 0, n_segments = 0, n_visits = 0, n_fast = 0;
    long long t_pack = 0, t_general = 0;      // cycles inside pack commands / the general first-fit loop (hqs_debug_read)
    // HQS_PATH_* bits of the header (hqs_stats.solver_path): where the solve's data lives, then the loops the solver warp ran
    u32 path = (a.sm.classes == SM_NONE ? HQS_PATH_CLASSES_GLOBAL : 0u) | (NARROW && a.sm.rem == SM_NONE ? HQS_PATH_REM_GLOBAL : 0u) |
               (glist_sm ? 0u : HQS_PATH_GROUPS_GLOBAL) | (a.blocked && a.sm.blocked == SM_NONE ? HQS_PATH_BLOCKED_GLOBAL : 0u) |
               ((a.x_world || a.before_ext) && a.sm.bef == SM_NONE ? HQS_PATH_COUNTS_GLOBAL : 0u);
#ifdef HQS_TRACE
    // measuring build (tools/trace_build.sh): cycle sums of the sections of the lean loop replace the phase stamps
    u32 tr_top = 0, tr_rec = 0, tr_cyc[4] = {0, 0, 0, 0}, tr_n[4] = {0, 0, 0, 0}, tr_fit = 0, tr_load = 0;   // visit kinds: dead tile, fall, scan (tile exhausted), scan (group ends)
#define TR_CLK() ([] { u32 c_; asm volatile("mov.u32 %0, %%clock;" : "=r"(c_)::"memory"); return c_; }())
#endif
    bool seg_overflow = false;
    if (warp != 0) {
        for (;;) {
            bar_named(1, TICK_THREADS);
            const u32 cmd = s_blk[0];
            if (cmd == BLK_END) break;
            block_work(cmd);
        }
    } else {
        const u32 lt_mask = (1u << lane) - 1;
        const bool resv_on = s_partial != 0;        // some worker is partly occupied at tick start: reservations are possible
        for (u32 pass = 0;; ++pass) {
            u32 seg_base = 0, out_base = 0;
            bool packed = (a.flags & TF_PACK) == 0;
            seg_overflow = false;
            u32 li = 0;
            while (li < n_list) {
                // ---- one priority level: entries [li, lj)
                const u32 lvl = s_gcl[li] >> 16;
                u32 lj = li + 1;
                for (;;) {
                    const u32 e = lj + lane;
                    const u32 m = __ballot_sync(0xffffffffu, e < n_list && (s_gcl[e] >> 16) == lvl);
                    if (m == 0xffffffffu) { lj += 32; continue; }
                    lj += (u32)__ffs(~m) - 1;
                    break;
                }
                const u32 ng = lj - li;
                bool level_packed = false;
                if (!packed && !skip_sat && ng <= PACK_MAX_CAND) {
                    // ---- is this level saturated?  demand (first variant of the tick's order) vs free, exact
                    //      saturating u64.  Lanes own entries li + lane, li + lane + 32.
                    u64 dem[RT], cap[RT];
                    u32 n_cand = 0, has_all = 0;
#pragma unroll
                    for (int r = 0; r < RT; ++r) { dem[r] = 0; cap[r] = 0; }
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const u32 e = li + lane + 32 * j;
                        if (e < lj) {
                            const u32 c = s_gcl[e] & 0xFFFFu, n = s_glist[e].y;
                            const u32 nvv = classes[c].n_variants;
                            n_cand += nvv;
                            for (u32 v = 0; v < nvv; ++v) has_all |= classes[c].v[v].all_mask ? 1u : 0u;
                            const Var& dv = classes[c].v[vorder[c * HQS_MAX_VARIANTS]];
                            bool servable = true;
#pragma unroll
                            for (int r = 0; r < RT; ++r) servable &= (u64)dv.amount[r] <= s_totmax[r];
                            if (servable) {
#pragma unroll
                                for (int r = 0; r < RT; ++r) dem[r] = sat_add64(dem[r], sat_mul64(exact_amount(dv, r), (u64)n));
                            }
                        }
                    }
                    for (u32 w = lane; w < W; w += 32) {
                        if (s_excl[w]) continue;
#pragma unroll
                        for (int r = 0; r < RT; ++r) cap[r] = sat_add64(cap[r], exact_of(s_fr[(size_t)w * RT + r], w, r));
                    }
#pragma unroll
                    for (int d = 16; d >= 1; d >>= 1) {
                        n_cand += __shfl_xor_sync(0xffffffffu, n_cand, d);
                        has_all |= __shfl_xor_sync(0xffffffffu, has_all, d);
#pragma unroll
                        for (int r = 0; r < RT; ++r) {
                            dem[r] = sat_add64(dem[r], __shfl_xor_sync(0xffffffffu, dem[r], d));
                            cap[r] = sat_add64(cap[r], __shfl_xor_sync(0xffffffffu, cap[r], d));
                        }
                    }
                    if (n_cand <= PACK_MAX_CAND && !has_all) {
                        // phi = the fraction of the level's demand the pool can serve, when two or more resources are
                        // over-subscribed (the classes then complement each other and each gets the same fraction of
                        // its demand this tick); with a single scarce resource any split drains at the same rate
                        u32 n_sat = 0;
                        double phi = 1.0;
#pragma unroll
                        for (int r = 0; r < RT; ++r)
                            if (r < (int)R && cap[r] != HQS_AMOUNT_MAX && dem[r] > cap[r]) n_sat++;
                        if (n_sat >= 2) {
#pragma unroll
                            for (int r = 0; r < RT; ++r)
                                if (r < (int)R && cap[r] != HQS_AMOUNT_MAX && dem[r] > 0) {
                                    const double x = __ddiv_rn(__ull2double_rn(cap[r]), __ull2double_rn(dem[r]));
                                    phi = x < phi ? x : phi;
                                }
                        }
                        if (n_sat != 0) {
                            if (lane == 0) {
                                s_blk[0] = BLK_PACK; s_blk[1] = li; s_blk[2] = lj; s_blk[3] = seg_base;
                                s_blk[4] = (u32)__double2loint(phi); s_blk[5] = (u32)__double2hiint(phi);
                            }
                            __syncwarp();
                            const long long tp0 = clock64();
                            bar_named(1, TICK_THREADS);
                            block_work(BLK_PACK);
                            t_pack += clock64() - tp0;
                            packed = true;
                            level_packed = s_err == 0;
                            if (level_packed) path |= HQS_PATH_PACKED;
                        }
                    }
                }
                if (plain && (packed || skip_sat) && !level_packed) {
                    // two instantiations of the same loop: without reservations and proactive filling (no worker is partly
                    // occupied at tick start, the usual M1 / zero-duration case) the bookkeeping for them is compiled out
                    auto lean_loop = [&](auto extras_tag) {
                        constexpr bool EXTRAS = decltype(extras_tag)::value;
                        // ---- lean first-fit over ALL remaining groups (no more packing can happen): the frontier tile's free
                        //      vectors stay in registers (lane = worker) from group to group, the next group's request is
                        //      prefetched, and the only work on the group-to-group dependency chain is fit -> ballot -> take.
                        u32 cur_tile = 0xFFFFFFFFu;
                        bool dirty = false, lane_excl = false;
                        AT fr[RT];
    #pragma unroll
                        for (int r = 0; r < RT; ++r) fr[r] = 0;
                        uint2 ge_n = s_glist[li];
                        u32 c_n = s_gcl[li] & 0xFFFFu;
                        Var dv_n = classes[c_n].v[0];
                        u32 front_n = s_front[c_n];
                        for (u32 e = li; e < n_list; ++e) {
#ifdef HQS_TRACE
                            const u32 tr0 = TR_CLK();
#endif
                            const uint2 ge = ge_n;
                            const u32 c = c_n;
                            Var dv = dv_n;
                            dv.all_mask = 0;                                         // plain tick: lets the compiler drop the `All` arm
                            const u32 tile0 = front_n >> 5;                         // s_front[c]: frontier WORKER (tile-granular here)
                            if (e + 1 < n_list) {
                                ge_n = s_glist[e + 1];
                                c_n = s_gcl[e + 1] & 0xFFFFu;
                                dv_n = classes[c_n].v[0];
                                front_n = s_front[c_n];
                            }
                            const u32 g = ge.x, n_all = ge.y;
                            u32 remaining = n_all, tile = tile0, f = tile0;
                            const u32 seg_lo = seg_base;
                            u32 seg_cur = seg_base;
                            bool front = true;
#ifdef HQS_TRACE
                            u32 tr1 = TR_CLK();
                            tr_top += tr1 - tr0;
#endif
                            while (remaining && tile < n_tiles) {
#ifdef HQS_TRACE
                                const u32 v0 = TR_CLK();
                                u32 kind = 0;
#endif
                                const u32 w = tile * 32 + lane;
                                if (tile != cur_tile) {
                                    if (dirty) {
                                        const u32 wo = cur_tile * 32 + lane;
                                        if (wo < W) {
    #pragma unroll
                                            for (int r = 0; r < RT; ++r) s_fr[(size_t)wo * RT + r] = fr[r];
                                        }
                                    }
    #pragma unroll
                                    for (int r = 0; r < RT; ++r) fr[r] = w < W ? s_fr[(size_t)w * RT + r] : 0;
                                    lane_excl = EXTRAS && resv_on && w < W && s_excl[w] != 0;   // reserved for a waiting class
                                    cur_tile = tile;
                                    dirty = false;
                                }
                                ++n_visits;
#ifdef HQS_TRACE
                                const u32 v1 = TR_CLK();
#endif
                                const u64 cnt = lane_excl ? 0 : fit_count<RT>(fr, 0u, dv, remaining);     // lanes beyond the pool hold zeros: 0
                                const u32 hasm = __ballot_sync(0xffffffffu, cnt != 0);
#ifdef HQS_TRACE
                                const u32 v2 = TR_CLK() + (hasm & 0);
#endif
                                u32 take = 0, exc = 0, handed = 0;
                                if (hasm) {
                                    const u32 first = (u32)__ffs(hasm) - 1;
                                    const u32 fall = __shfl_sync(0xffffffffu, cnt >= remaining ? 1u : 0u, first);
                                    if (fall) {
#ifdef HQS_TRACE
                                        kind = 1;
#endif
                                        take = lane == first ? remaining : 0;
                                        handed = remaining;
                                    } else if (remaining <= 0x03FFFFFFu) {
                                        u32 inc = (u32)cnt;
    #pragma unroll
                                        for (int d = 1; d < 32; d <<= 1) {
                                            const u32 y = __shfl_up_sync(0xffffffffu, inc, d);
                                            if ((int)lane >= d) inc += y;
                                        }
                                        exc = inc - (u32)cnt;
                                        if (cnt && exc < remaining) take = min((u32)cnt, remaining - exc);
                                        const u32 total = __shfl_sync(0xffffffffu, inc, 31);
                                        handed = min(total, remaining);
#ifdef HQS_TRACE
                                        kind = total < remaining ? 2 : 3;
#endif
                                    } else {
                                        u64 inc = cnt;
    #pragma unroll
                                        for (int d = 1; d < 32; d <<= 1) {
                                            const u64 y = __shfl_up_sync(0xffffffffu, inc, d);
                                            if ((int)lane >= d) inc += y;
                                        }
                                        const u64 e64 = inc - cnt;
                                        exc = (u32)(e64 < remaining ? e64 : remaining);
                                        if (cnt && e64 < remaining) take = (u32)(cnt < remaining - e64 ? cnt : remaining - e64);
                                        const u64 total = __shfl_sync(0xffffffffu, inc, 31);
                                        handed = (u32)(total < remaining ? total : remaining);
                                    }
                                }
                                const u32 tkm = __ballot_sync(0xffffffffu, take != 0);
                                if (take) {
                                    const u32 si = seg_cur + __popc(tkm & lt_mask);
                                    if (si < SEG_CAP) { a.seg_cum[si] = (n_all - remaining) + exc + take; a.seg_wv[si] = w; }
                                }
                                take_from<RT, AT>(fr, dv, take);                       // take == 0 leaves the lane as it is
                                if (EXTRAS && resv_on && take) s_touch[w] = 1;
                                dirty |= tkm != 0;
                                seg_cur += __popc(tkm);
                                if (front) {
                                    const u32 alive = __ballot_sync(0xffffffffu, !(cnt < remaining && take == (u32)cnt));
                                    if (alive == 0) f = tile + 1; else front = false;
                                }
                                remaining -= handed;
                                if (remaining) ++tile;
#ifdef HQS_TRACE
                                {
                                    const u32 v3 = TR_CLK() + (remaining & 0);
                                    tr_load += v1 - v0; tr_fit += v2 - v1;
                                    if (kind == 0) { tr_cyc[0] += v3 - v0; ++tr_n[0]; }
                                    if (kind == 1) { tr_cyc[1] += v3 - v0; ++tr_n[1]; }
                                    if (kind == 2) { tr_cyc[2] += v3 - v0; ++tr_n[2]; }
                                    if (kind == 3) { tr_cyc[3] += v3 - v0; ++tr_n[3]; }
                                }
#endif
                            }
#ifdef HQS_TRACE
                            const u32 tr3 = TR_CLK() + (remaining & 0);
#endif
                            if (f != tile0 && lane == 0) s_front[c] = (unsigned short)(f * 32);
                            if (c_n == c && f != tile0) front_n = f * 32;            // the same class again (next level)
                            if (EXTRAS && resv_on && remaining && !s_noresv[c]) {
                                // the class is left with unplaced tasks: reservations.  The tile in registers goes back first
                                // and is loaded again afterwards (with the new exclusions)
                                if (dirty) {
                                    const u32 wo = cur_tile * 32 + lane;
                                    if (wo < W) {
    #pragma unroll
                                        for (int r = 0; r < RT; ++r) s_fr[(size_t)wo * RT + r] = fr[r];
                                    }
                                    dirty = false;
                                }
                                __syncwarp();
                                reserve_for(c, n_all, remaining);
                                cur_tile = 0xFFFFFFFFu;
                            }
                            const u32 k = n_all - remaining;
                            if (EXTRAS && s_kk && lane == 0) s_kk[e] = k;
                            u32 k_loc = k;
                            if (before) {
                                const u32 bef = s_bef ? s_bef[e] : __ldcg(before + g);
                                const u32 loc = s_loc ? s_loc[e] : __ldcg(a.total_local + g);
                                k_loc = k > bef ? k - bef : 0;
                                k_loc = k_loc < loc ? k_loc : loc;
                            }
                            if (lane == 0) {
                                GroupOut go;
                                go.k = k; go.out_off = out_base; go.seg_lo = seg_lo; go.seg_n = seg_cur - seg_lo;
                                a.gout[g] = go;
                            }
                            out_base += k_loc;
                            seg_base = seg_cur;
                            if (seg_base > SEG_CAP) { seg_overflow = true; seg_base = SEG_CAP; }
#ifdef HQS_TRACE
                            tr_rec += TR_CLK() + (out_base & 0) - tr3;
#endif
                        }
                        if (dirty) {
                            const u32 wo = cur_tile * 32 + lane;
                            if (wo < W) {
    #pragma unroll
                                for (int r = 0; r < RT; ++r) s_fr[(size_t)wo * RT + r] = fr[r];
                            }
                        }
                    };
                    if (resv_on || s_kk) { lean_loop(std::true_type{}); path |= HQS_PATH_LEAN_EXTRAS; }
                    else if (wide_ok) {
                        path |= HQS_PATH_WIDE;
                        // every worker a lane: all warps of the CTA (see wide_loop)
                        if (lane == 0) { s_blk[0] = BLK_WIDE; s_blk[1] = li; s_blk[2] = out_base; s_blk[3] = seg_base; }
                        __syncwarp();
                        bar_named(1, TICK_THREADS);
                        const WideOut wo = run_wide();
                        seg_base = wo.seg_base; out_base = wo.out_base;
                        seg_overflow |= wo.overflow;
                        n_visits += wo.steps;
                    } else { lean_loop(std::false_type{}); path |= HQS_PATH_LEAN; }
                    __syncwarp();
                    n_fast += n_list - li;
                    li = n_list;
                    break;
                }
                // ---- the groups of the level, in order: first-fit (after what pack placed)
                const long long tg0 = clock64();
                path |= HQS_PATH_GENERAL;
                u32 region_end = seg_base;
                if (level_packed) {
                    region_end = seg_base + 2u * W * s_cbase[ng];
                    if (region_end > SEG_CAP) { seg_overflow = true; }
                }
                for (u32 e = li; e < lj; ++e) {
                    const uint2 ge = s_glist[e];
                    const u32 g = ge.x, n_all = ge.y;
                    const u32 c = s_gcl[e] & 0xFFFFu;
                    const Cls& cl = classes[c];
                    const u32 nv = cl.n_variants;
                    u32 remaining = n_all;
                    u32 seg_lo = seg_base, seg_cur = seg_base;
                    if (level_packed) {
                        seg_lo = s_pkseglo[e - li];
                        seg_cur = seg_lo + s_pknseg[e - li];
                        remaining = n_all - s_pkpos[e - li];
                        // hand back what the workers took beyond the class count (tiles [ex_lo, ex_hi))
                        const u32 ex_lo = s_pkex[e - li] & 0xFFFFu, ex_hi = s_pkex[e - li] >> 16;
                        if (ex_lo < ex_hi) {
                            for (u32 tile = ex_lo; tile < ex_hi; ++tile) {
                                const u32 w = tile * 32 + lane;
                                for (u32 v = 0; v < nv; ++v) {
                                    const u32 ex = w < W ? __ldcg(a.pk.taken + (size_t)w * PACK_MAX_CAND + s_cbase[e - li] + v) : 0;
                                    if (!ex) continue;
                                    const Var& dv = cl.v[v];
#pragma unroll
                                    for (int r = 0; r < RT; ++r)
                                        if (((dv.used_mask >> r) & 1) && s_fr[(size_t)w * RT + r] != AMAX)
                                            s_fr[(size_t)w * RT + r] += (AT)((u64)ex * dv.amount[r]);
                                }
                            }
                            // free amounts grew: no frontier may lie beyond the first tile that got something back
                            for (u32 c2 = lane; c2 < Q; c2 += 32)
                                if (s_front[c2] > ex_lo * 32) s_front[c2] = (unsigned short)(ex_lo * 32);
                            __syncwarp();
                        }
                    }
                    for (u32 vi = 0; vi < nv && remaining; ++vi) {
                        // Each worker offers the untried variant that costs the smallest share of what it has left:
                        // min over variants of max_r f32(amount_r) * (1 / f32(free_r)), `All` = +inf, ties to the lower
                        // variant id (specification: tests/greedy_model.py::_Tick.next_variant).
                        const bool last_round = vi + 1 == nv;
                        bool front = true;
                        for (u32 tile = s_front[c] >> 5; tile < n_tiles && remaining; ++tile) {
                            ++n_visits;
                            const u32 w = tile * 32 + lane;
                            const bool in_pool = w < W;
                            const bool has = in_pool && !s_excl[w];
                            AT fr[RT];
#pragma unroll
                            for (int r = 0; r < RT; ++r) fr[r] = in_pool ? s_fr[(size_t)w * RT + r] : 0;
                            const u32 unt = in_pool ? s_unt[w] : 0;
                            u32 v = 0, td = 0;
                            if (nv > 1) {
                                td = (vi && in_pool) ? s_td[w] : 0;
                                float inv[RT];
#pragma unroll
                                for (int r = 0; r < RT; ++r)
                                    inv[r] = __fdiv_rn(1.0f, __double2float_rn(__ull2double_rn(in_pool ? exact_of(fr[r], w, r) : 0)));
                                float best_d = 0.0f;
                                int best_v = -1;
                                for (u32 vv = 0; vv < nv; ++vv) {
                                    if ((td >> vv) & 1) continue;
                                    const Var& cv = cl.v[vv];
                                    float dom = 0.0f;
                                    if (cv.all_mask) dom = __int_as_float(0x7f800000);
                                    else {
#pragma unroll
                                        for (int r = 0; r < RT; ++r) {
                                            if (!((cv.used_mask >> r) & 1) || fr[r] == AMAX) continue;
                                            const float x = __fmul_rn(cv.rcpf[RT + r], inv[r]);
                                            dom = x > dom ? x : dom;
                                        }
                                    }
                                    if (best_v < 0 || dom < best_d) { best_v = (int)vv; best_d = dom; }
                                }
                                v = (u32)best_v;
                            }
                            const Var& dv = cl.v[v];
                            u64 cnt = 0;
                            if (has) {
                                const uint8_t blk = blocked ? blocked[(size_t)w * Q + c] : 0;
                                const u64 rt = a.any_time_limit ? s_remtime[w] : HQS_TIME_INF;
                                if (admissible(dv, v, blk, rt)) cnt = fit_count<RT>(fr, unt, dv, remaining);
                            }
                            // ---- hand out `remaining` in worker order: the first worker that can take anything often
                            //      takes it all (mode M1); otherwise an inclusive scan over the tile
                            const u32 hasm = __ballot_sync(0xffffffffu, cnt != 0);
                            if (hasm == 0 && nv == 1) {                  // a dead tile (one variant: nothing to record per worker)
                                if (front && lane == 0) s_front[c] = (unsigned short)((tile + 1) * 32);
                                __syncwarp();
                                continue;
                            }
                            u32 take = 0, exc = 0, handed = 0;
                            if (hasm) {
                                const u32 first = (u32)__ffs(hasm) - 1;
                                const u32 fall = __shfl_sync(0xffffffffu, cnt >= remaining ? 1u : 0u, first);
                                if (fall) {
                                    take = lane == first ? remaining : 0;
                                    handed = remaining;
                                } else if (remaining <= 0x03FFFFFFu) {
                                    u32 inc = (u32)cnt;
#pragma unroll
                                    for (int d = 1; d < 32; d <<= 1) {
                                        const u32 y = __shfl_up_sync(0xffffffffu, inc, d);
                                        if ((int)lane >= d) inc += y;
                                    }
                                    exc = inc - (u32)cnt;
                                    if (cnt && exc < remaining) take = min((u32)cnt, remaining - exc);
                                    const u32 total = __shfl_sync(0xffffffffu, inc, 31);
                                    handed = min(total, remaining);
                                } else {
                                    u64 inc = cnt;
#pragma unroll
                                    for (int d = 1; d < 32; d <<= 1) {
                                        const u64 y = __shfl_up_sync(0xffffffffu, inc, d);
                                        if ((int)lane >= d) inc += y;
                                    }
                                    const u64 e64 = inc - cnt;
                                    exc = (u32)(e64 < remaining ? e64 : remaining);
                                    if (cnt && e64 < remaining) take = (u32)(cnt < remaining - e64 ? cnt : remaining - e64);
                                    const u64 total = __shfl_sync(0xffffffffu, inc, 31);
                                    handed = (u32)(total < remaining ? total : remaining);
                                }
                            }
                            const u32 tkm = __ballot_sync(0xffffffffu, take != 0);
                            if (take) {
                                const u32 si = seg_cur + __popc(tkm & lt_mask);
                                if (si < SEG_CAP) { a.seg_cum[si] = (n_all - remaining) + exc + take; a.seg_wv[si] = w | (v << 16); }
                                take_from<RT, AT>(fr, dv, take);
#pragma unroll
                                for (int r = 0; r < RT; ++r) s_fr[(size_t)w * RT + r] = fr[r];
                                // touched resources are no longer "untouched" (free == total); an unbounded amount stays as it is
                                u32 touched = dv.all_mask & dv.used_mask;
#pragma unroll
                                for (int r = 0; r < RT; ++r)
                                    if (((dv.used_mask >> r) & 1) && !((dv.all_mask >> r) & 1) && fr[r] != AMAX) touched |= 1u << r;
                                s_unt[w] = unt & ~touched;
                                s_touch[w] = 1;
                                if constexpr (NARROW) {
                                    // `All` consumed the whole resource: the exact free amount is 0, remainder included
                                    const u32 z = dv.all_mask & dv.used_mask;
                                    if (z) {
#pragma unroll
                                        for (int r = 0; r < RT; ++r)
                                            if ((z >> r) & 1) p_rem[(size_t)w * RT + r] = 0;
                                    }
                                }
                            }
                            seg_cur += __popc(tkm);
                            // ---- frontier: a worker whose fit count was not capped by `remaining` and that took all of it
                            //      has no room left for this variant; free amounts only shrink during first-fit
                            const bool dead_v = cnt < remaining && take == (u32)cnt;
                            bool lane_dead;
                            if (nv > 1) {
                                td |= (1u << v) | (dead_v ? (0x100u << v) : 0u);
                                if (in_pool) s_td[w] = (unsigned short)td;
                                lane_dead = last_round && (td >> 8) == ((1u << nv) - 1u);
                            } else {
                                lane_dead = dead_v;
                            }
                            if (front) {
                                const u32 alive = __ballot_sync(0xffffffffu, in_pool && !lane_dead);
                                if (alive == 0 && last_round) { if (lane == 0) s_front[c] = (unsigned short)((tile + 1) * 32); }
                                else front = false;
                            }
                            remaining -= handed;
                            __syncwarp();
                        }
                    }
                    if (resv_on && remaining && !s_noresv[c]) reserve_for(c, n_all, remaining);
                    const u32 k = n_all - remaining;
                    if (s_kk && lane == 0) s_kk[e] = k;
                    // local share of the k assigned tasks (sharded mode: ranks are ordered by handle range)
                    u32 k_loc = k;
                    if (before) {
                        const u32 bef = s_bef ? s_bef[e] : __ldcg(before + g);
                        const u32 loc = s_loc ? s_loc[e] : __ldcg(a.total_local + g);
                        k_loc = k > bef ? k - bef : 0;
                        k_loc = k_loc < loc ? k_loc : loc;
                    }
                    if (lane == 0) {
                        GroupOut go;
                        go.k = k; go.out_off = out_base; go.seg_lo = seg_lo; go.seg_n = seg_cur - seg_lo;
                        a.gout[g] = go;
                    }
                    out_base += k_loc;
                    if (!level_packed) {
                        seg_base = seg_cur;
                        if (seg_base > SEG_CAP) { seg_overflow = true; seg_base = SEG_CAP; }
                    }
                }
                if (level_packed) seg_base = region_end > SEG_CAP ? SEG_CAP : region_end;
                t_general += clock64() - tg0;
                li = lj;
            }
            n_assigned = out_base;
            n_segments = seg_base;
            // ---- min-utilisation (solver.rs:154-156, 479-518): a worker either receives at least
            //      min_cpus = total * (mu - 1) + free cpus of new work in this tick, or nothing.  The MILP has a boolean
            //      per worker; here a violating worker is taken out of the tick and the solve starts over, so its tasks
            //      go to the other workers (or stay ready).
            if (!a.min_util || pass + 1 >= MU_MAX_PASSES) break;
            u32 viol = 0;
            for (u32 w = lane; w < W; w += 32) {
                if (s_excl[w]) continue;
                const float muf = a.min_util[w];
                const u64 t0 = a.total_rw[(size_t)w * R], f0 = a.free_rw[(size_t)w * R];
                if (!(muf > 0.001f) || t0 == HQS_AMOUNT_MAX || f0 == HQS_AMOUNT_MAX) continue;
                const double mu = (double)muf;
                const double cpu_total = __ddiv_rn(__ull2double_rn(t0), 10000.0), cpu_free = __ddiv_rn(__ull2double_rn(f0), 10000.0);
                const double min_cpus = __dadd_rn(__dmul_rn(cpu_total, __dsub_rn(mu, 1.0)), cpu_free);
                const u64 fa = exact_of(s_fr[(size_t)w * RT + 0], w, 0);
                const double new_cpus = __ddiv_rn(__ull2double_rn(f0 - fa), 10000.0);
                if (min_cpus >= 0.0001 && new_cpus > 0.0 && new_cpus < __dsub_rn(min_cpus, 1e-9)) { s_excl[w] = 1; viol = 1; }
            }
            if (!__any_sync(0xffffffffu, viol)) break;
            // every listed group rewrites its record in the next pass
            path |= HQS_PATH_MU_RESTART;
            if (lane == 0) s_blk[0] = BLK_RESTART;
            __syncwarp();
            bar_named(1, TICK_THREADS);
            block_work(BLK_RESTART);
        }
        u32 n_prefilled = 0;
        if (a.pf_shift && a.pf_max && (a.flags & TF_EMIT)) {
            if (lane == 0) s_blk[0] = BLK_PREFILL;
            __syncwarp();
            bar_named(1, TICK_THREADS);
            block_work(BLK_PREFILL);
            n_prefilled = s_blk[7];
        }
        if (lane == 0) s_blk[0] = BLK_END;
        __syncwarp();
        // ---- release the worker CTAs as early as possible: they need the group records, the segments and n_segments
        u32 err = s_err ? 2u : s_xmis ? 4u : (seg_overflow ? 1u : 0u);
        if (!err && n_assigned + n_prefilled > a.out_cap && (a.flags & TF_EMIT)) err = 3u;
        if (err == 0 && (a.flags & TF_EMIT) && a.emit_stage && n_prefilled == 0) path |= HQS_PATH_EMIT_STAGED;     // as do_emit decides
        if (lane == 0) {
            a.hdr->n_segments = n_segments;
            a.hdr->n_assigned = n_assigned;
            a.hdr->n_prefilled = n_prefilled;
            a.hdr->error = err;
            s_npref = n_prefilled;
            __threadfence();
            const u32 seq = s_npacks + 1;
#ifdef HQS_TRACE
            s_trel = global_timer_ns();
#endif
            st_release(&a.sync->cmd, (seq << 2) | ((err == 0 && (a.flags & TF_EMIT)) ? CMD_EMIT : CMD_EXIT));
            s_final_err = err;
        }
        __syncwarp();
        bar_named(1, TICK_THREADS);
    }
    // ---- epilogue (all warps): free vectors after the tick, header, reset of the per-tick counters
    const long long t_solved = clock64();
    __syncthreads();
    for (u32 w = tid; w < W; w += blockDim.x) {
#pragma unroll
        for (int r = 0; r < RT; ++r)
            if (r < (int)R) {
                const u64 x = exact_of(s_fr[(size_t)w * RT + r], w, r);
                a.free_after[(size_t)w * R + r] = x;
                if (a.hdr_host) reinterpret_cast<u64*>(a.hdr_host + 1)[(size_t)w * R + r] = x;
            }
    }
#ifdef HQS_TRACE
    __syncthreads();
    const unsigned long long tr_fv = global_timer_ns();     // free vectors written (device copy and pinned host mirror)
#endif
    if (tid == 0) {
        if (!spin_until_ge(&a.sync->emit_done, nW)) s_err = 24;
    }
    __syncthreads();
    const long long t_end = clock64();
#ifdef HQS_TRACE
    const unsigned long long tr_seen = global_timer_ns();   // the solver CTA saw every worker CTA's emit_done
#endif
    for (u32 g = tid; g < G; g += blockDim.x) a.total_local[g] = 0;
    if (tid == 0) {
        u32 err = s_final_err;
        const u32 werr = __ldcg(&a.sync->error);
        if (!err && (s_err || werr)) err = 2u;
        TickHeaderOut h;
        h.n_assigned = warp == 0 ? n_assigned : 0;
        h.n_groups = n_list;
        h.n_segments = n_segments;
        h.error = err;
        h.n_prefilled = s_npref;
        h.pad = s_err ? s_err : (werr ? 25u : 0u);       // which wait timed out (21 histogram, 22 | peer << 8, 23 pack, 24 emit, 25 a worker CTA)
        h.solver_path = path;
        h.pad2 = s_xmis;                                  // detail of error 4: which peer, and its G
        h.dbg[0] = (unsigned long long)(t_counted - t_start);     // staging + wait for the histogram
        h.dbg[1] = (unsigned long long)(t_prologue - t_counted);  // exchange + compaction + demand
        h.dbg[2] = (unsigned long long)(t_solved - t_prologue);   // the solver warp
        h.dbg[3] = (unsigned long long)(t_end - t_solved);        // emit (+ free vectors)
        // groups (16 bits) | cycles / 256 inside the general first-fit loop (16 bits) | tile visits
        h.dbg[4] = (unsigned long long)(n_list & 0xFFFFu) | ((unsigned long long)((t_general >> 8) & 0xFFFF) << 16) | ((unsigned long long)n_visits << 32);
        h.dbg[5] = (unsigned long long)(t_end - t_start);
        h.dbg[6] = global_timer_ns() - gt_start;                  // the same interval in ns
        // pack commands (8 bits) | cycles / 256 inside them (24 bits) | groups of the lean loop
        h.dbg[7] = (unsigned long long)(s_npacks & 0xFFu) | ((unsigned long long)((t_pack >> 8) & 0xFFFFFF) << 8) | ((unsigned long long)n_fast << 32);
#ifdef HQS_TRACE
        h.dbg[0] = ((unsigned long long)tr_rec << 32) | tr_top;
        h.dbg[1] = ((unsigned long long)tr_fit << 32) | tr_load;
        for (int q = 0; q < 4; ++q) h.dbg[2 + q] = ((unsigned long long)tr_n[q] << 32) | tr_cyc[q];
        h.dbg[6] = (unsigned long long)(t_solved - t_prologue);
        // emit tail, 16-bit fields in units of 16 ns after the release of the grid's last command (tools/trace_emit.py):
        // dbg[7] = worker CTAs (maxima): command seen | staged | chunk filter | emit_finish;
        // dbg[5] (wide loop) = emit_done counted | solver CTA: free vectors written | every emit_done seen | worker CTAs with work
        auto d16 = [&](unsigned long long t) -> unsigned long long {
            const unsigned long long d = t > s_trel ? (t - s_trel) >> 4 : 0;
            return d < 0xFFFFu ? d : 0xFFFFu;
        };
        unsigned long long te[6];
        for (int q = 0; q < 6; ++q) { te[q] = __ldcg(&a.sync->tr_emit[q]); a.sync->tr_emit[q] = 0; }
        h.dbg[7] = d16(te[TR_EMIT_CMD]) | (d16(te[TR_EMIT_STAGED]) << 16) | (d16(te[TR_EMIT_FILTER]) << 32) | (d16(te[TR_EMIT_FINISH]) << 48);
        if (n_fast && tr_n[0] + tr_n[1] + tr_n[2] + tr_n[3] == 0) {      // the wide loop ran: its section sums (warp 0)
            for (int q = 0; q < 4; ++q) h.dbg[q] = ((unsigned long long)s_trw[2 * q + 1] << 32) | s_trw[2 * q];
            h.dbg[4] = n_visits;
            h.dbg[5] = d16(te[TR_EMIT_DONE]) | (d16(tr_fv) << 16) | (d16(tr_seen) << 32) |
                       ((te[TR_EMIT_NWORK] < 0xFFFFu ? te[TR_EMIT_NWORK] : 0xFFFFu) << 48);
        }
#endif
        *a.hdr = h;
        if (a.hdr_host) *a.hdr_host = h;
        // the tick is over: every worker CTA has left its loops
        a.sync->cmd = 0; a.sync->count_done = 0; a.sync->scan_done = 0; a.sync->pack_done = 0; a.sync->emit_done = 0;
        a.sync->error = 0;
        __threadfence_system();
    }
}

template <int RT, typename AT>
__global__ void __launch_bounds__(TICK_THREADS, 1) tick_k(const __grid_constant__ TickArgs a) {
    extern __shared__ __align__(16) unsigned char smem_dyn[];
    if (blockIdx.x == 0) solver_cta<RT, AT>(a, smem_dyn);
    else worker_cta<RT>(a, smem_dyn);
}

// standalone histogram (NCCL variant of the sharded tick: the host all-gathers the totals between the two halves)
__global__ void __launch_bounds__(TICK_THREADS) count_only_k(const __grid_constant__ TickArgs a) {
    extern __shared__ __align__(16) unsigned char smem_dyn[];
    for (u32 b = blockIdx.x; b < a.P; b += gridDim.x) count_chunk(a, b, reinterpret_cast<u32*>(smem_dyn));
}

// per-worker totals of the count segments (what-if query)
__global__ void seg_worker_totals_k(const GroupOut* __restrict__ gout, u32 G, const u32* __restrict__ seg_cum,
                                    const u32* __restrict__ seg_wv, u32* __restrict__ per_worker) {
    // one thread per group: walks the group's segments (inclusive end ranks -> counts)
    const u32 g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const GroupOut go = gout[g];
    if (go.k == 0) return;
    u32 prev = 0;
    for (u32 i = 0; i < go.seg_n; ++i) {
        const u32 end = seg_cum[go.seg_lo + i];
        atomicAdd(&per_worker[seg_wv[go.seg_lo + i] & 0xFFFFu], end - prev);
        prev = end;
    }
}
