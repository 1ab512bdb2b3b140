/*
 * hqsched.h — C ABI of the H100-native (sm_90a) task->worker assignment solver (libhqsched_b200.so).
 *
 * Drop-in boundary for the hot path of HyperQueue's tako scheduler tick (v0.26.0).  The reference has
 * no FFI for this path; the seam it replaces is the pair
 *     run_scheduling_solver()   crates/tako/src/internal/scheduler/solver.rs:16-461
 *     create_task_mapping()     crates/tako/src/internal/scheduler/mapping.rs:23-154  (task selection half)
 * called from run_scheduling_inner()  crates/tako/src/internal/scheduler/main.rs:40-46.
 * A Rust shim (INTEGRATION.md) keeps Core mutation and Comm::send_worker_message in Rust and calls
 * this library through bindgen, the same way `highs-sys` binds HiGHS today (Cargo.lock:1116-1123).
 *
 * Conventions
 *  - plain C, no exceptions / longjmp across the ABI, caller-owned host buffers (pinned or pageable),
 *  - every function returns 0 on success and a negative HQS_E_* code on failure; after a failed
 *    hqs_tick the host must schedule NOTHING this tick (mirrors "solver returned None => empty
 *    solution", solver.rs:412-415) and the device has consumed nothing either: the ready set is as it was
 *    before the call (HQS_E_OVERFLOW, HQS_E_LIMIT: the solver decides before anything is emitted);
 *    hqs_last_error() gives the text,
 *  - called from tako's single reactor thread; a context is not thread-safe,
 *  - tasks are named by dense u32 handles chosen by the shim IN TaskId ORDER (ascending handle ==
 *    ascending (job_id, job_task_id)), because the ready set is popped in ascending TaskId inside one
 *    priority level (scheduler/taskqueue.rs:395-420) and the device ranks tasks by handle,
 *  - amounts are ResourceAmount fractions (u64, 10 000 per unit, common/resources/amount.rs:7,26);
 *    ~0 is ResourceAmount::MAX ("unknown/unbounded", amount.rs:30),
 *  - priorities are tako Priority values (u64, larger = more urgent, common/priority.rs:36-48).
 */
#ifndef HQSCHED_H
#define HQSCHED_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HQS_ABI_VERSION 1
#define HQS_MAX_RESOURCES 16u   /* resource kinds per context (R)                                  */
#define HQS_MAX_VARIANTS 8u     /* variants per request class (reference allows 32, request.rs:305) */
#define HQS_MAX_WORKERS 1024u   /* workers per tick (one solver thread per worker)                  */
#define HQS_MAX_CLASSES 4096u   /* interned request classes (ResourceRqId)                          */
#define HQS_MAX_GROUPS 8192u    /* (priority level x class) groups of LIVE levels; more: levels are merged */
#define HQS_AMOUNT_MAX (~(uint64_t)0)
#define HQS_TIME_INF (~(uint64_t)0)

enum {
    HQS_OK = 0,
    HQS_E_INVALID = -1,   /* bad argument                                   */
    HQS_E_CUDA = -2,      /* CUDA runtime error (text in hqs_last_error)    */
    HQS_E_LIMIT = -3,     /* a compile-time limit above was exceeded        */
    HQS_E_NOMEM = -4,
    HQS_E_OVERFLOW = -5,  /* out_cap too small for the assignments produced */
    HQS_E_STATE = -6      /* call sequence error                            */
};

typedef struct hqs_ctx hqs_ctx;

/* One variant of a request class = ResourceRequest (common/resources/request.rs:136-167) in dense
 * per-resource form.  amount[r] == 0: resource r not requested.  Bit r of all_mask: policy `All`
 * (request.rs:20): needs >= 1 fraction free to be feasible and consumes the worker's TOTAL of r
 * (solver.rs:120-124).  The five amount policies (compact/tight/scatter/forced) are identical on the
 * server side (request.rs:38-48) and are not distinguished here. */
typedef struct {
    uint64_t amount[HQS_MAX_RESOURCES];
    uint32_t all_mask;
    uint32_t weight;        /* ResourceWeight raw value, 10 000 = 1.0 (request.rs:107-134) */
    uint64_t min_time_ms;   /* TimeRequest (request.rs:143-149) in milliseconds            */
} hqs_variant;

/* ResourceRequestVariants (request.rs:229-316), interned as ResourceRqId = index in the array given
 * to hqs_classes_set (common/resources/map.rs:99-109).  n_nodes > 0 (multi-node) is rejected:
 * multi-node placement is outside this path (SURVEY.md §8(f) row 4). */
typedef struct {
    uint32_t n_variants;
    uint32_t n_nodes;
    hqs_variant variants[HQS_MAX_VARIANTS];
} hqs_class;

/* Server-side view of one worker for one tick (server/worker.rs:63-84).  The array passed to
 * hqs_tick must be sorted by ascending worker_id (solver.rs:44). */
typedef struct {
    uint32_t worker_id;
    uint32_t flags;              /* reserved, 0                                                   */
    uint64_t remaining_time_ms;  /* termination_time - now, HQS_TIME_INF if none (worker.rs:320)   */
    float min_utilization;       /* WorkerConfiguration::min_utilization (solver.rs:154-156, 479-518): enforced by
                                    the tick — the worker gets at least total*(mu-1)+free cpus of new work or nothing */
    uint32_t reserved;
} hqs_worker;

/* One emitted placement.  8 bytes: the unit of the output stream. */
typedef struct {
    uint32_t task;     /* handle                                                         */
    uint16_t worker;   /* INDEX into the workers[] array of this tick (not worker_id)    */
    uint8_t variant;   /* ResourceVariantId                                              */
    uint8_t kind;      /* 0 = assign (ComputeTasks with the variant)
                          1 = prefill (ComputeTasks with variant = None, mapping.rs:156-230): the task stays ready
                          2 = the task was prefilled on another worker: RetractTasks to that worker (the host knows
                              which) + redirect to `worker` / `variant` (mapping.rs:63-101)                   */
} hqs_assignment;

typedef struct {
    uint32_t n_groups;          /* non-empty (priority level, class) groups seen by the last tick */
    uint32_t n_levels;          /* priority levels (after coarsening)                             */
    uint32_t n_assigned;        /* assignments produced by the last tick                          */
    uint32_t n_segments;        /* (group, worker, variant) count segments of the last tick       */
    uint64_t kernel_launches;   /* kernels launched by this context so far                        */
    uint64_t ticks;
    uint32_t n_handles;         /* size of the device task table                                  */
    uint32_t coarsened;         /* 1 if LIVE priority levels had to be merged to fit HQS_MAX_GROUPS: tasks of merged
                                   levels are then ordered by class and handle, not by priority — log it         */
    uint32_t narrow_amounts;    /* 1 if the last tick solved on gcd-scaled 32-bit amounts          */
    uint32_t solver_path;       /* HQS_PATH_* bits: how the last tick (or query) solved            */
} hqs_stats;

/* hqs_stats.solver_path.  The first four bits name the first-fit loops that ran (several can, one after the other:
 * packed levels are followed by the general loop, a minimum-utilisation restart runs the solve again). */
#define HQS_PATH_WIDE 0x01u            /* wide loop: every worker of a pool of <= 512 is a lane               */
#define HQS_PATH_LEAN 0x02u            /* one-warp lean loop (plain tick)                                     */
#define HQS_PATH_LEAN_EXTRAS 0x04u     /* lean loop with reservation / proactive-filling bookkeeping          */
#define HQS_PATH_GENERAL 0x08u         /* general loop (variants, `All`, blocked masks, time limits, packing) */
#define HQS_PATH_PACKED 0x10u          /* at least one saturated priority level was packed                    */
#define HQS_PATH_MU_RESTART 0x20u      /* the minimum-utilisation rule restarted the solve                    */
#define HQS_PATH_CLASSES_GLOBAL 0x40u  /* the class table did not fit shared memory and was read from global  */
#define HQS_PATH_REM_GLOBAL 0x80u      /* narrow remainders did not fit shared memory and live in global       */
#define HQS_PATH_EMIT_STAGED 0x100u    /* the tick emitted each chunk's assignments as per-group runs staged in shared
                                          memory; clear on an emitting tick: one pass per task (large group counts,
                                          ticks with prefill records, HQS_DEBUG_EMIT_PER_TASK; in a sharded tick this
                                          is the rank's own prefill records, so the bit can differ between ranks)  */
#define HQS_PATH_GROUPS_GLOBAL 0x200u  /* the solver's group list did not fit shared memory next to the worker state (many
                                          workers x wide amounts x thousands of groups) and lives in global memory    */
#define HQS_PATH_BLOCKED_GLOBAL 0x400u /* the blocked mask did not fit shared memory and was read from global          */
#define HQS_PATH_COUNTS_GLOBAL 0x800u  /* sharded tick: the per-group counts of this rank and of the lower ranks did not
                                          fit shared memory and were read from global                                  */

int hqs_abi_version(void);

/* Creates a context on CUDA device `device`.  n_resources = number of resource kinds (R <= 16).
 * flags: bit 0 = no packing of the first saturated priority level (plain first-fit everywhere);
 *        bit 1 = always solve on 64-bit amounts (default: amounts are divided by the per-resource gcd of
 *                the requested amounts and solved in 32 bits whenever every scaled amount of the tick is
 *                below 2^31 — same results, shorter critical path).  Both bits exist for tests. */
#define HQS_CREATE_NO_PACK 1u
#define HQS_CREATE_WIDE_AMOUNTS 2u
/*        bit 2 = the tick kernel occupies half of the SMs only, so that two contexts whose ticks wait for each other on
 *                the device (peer exchange between two contexts of one GPU) can run side by side. */
#define HQS_CREATE_SHARE_DEVICE 4u
int hqs_create(hqs_ctx** out, int device, uint32_t n_resources, uint32_t flags);
void hqs_destroy(hqs_ctx* ctx);
const char* hqs_last_error(const hqs_ctx* ctx);   /* ctx may be NULL: last error of hqs_create */

/* Replaces the class table (mirror of ResourceRqMap; ids are array indices, append-only in tako). */
int hqs_classes_set(hqs_ctx* ctx, uint32_t n_classes, const hqs_class* classes);

/* TaskQueues::add_ready_task (taskqueue.rs:37-43) for n tasks: the task becomes ready with the given
 * class and priority.  Handles may be new or re-used after the task left the ready set. */
int hqs_ready_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id,
                   const uint64_t* priority);
/* The same for a task array: the handles are first_task .. first_task + n - 1 (tako's job arrays are consecutive
 * TaskIds, so the shim's handles are too) and no handle array crosses PCIe.  A batch with an invalid class id is
 * rejected as a whole (validated on the device before the table is touched). */
int hqs_ready_push_range(hqs_ctx* ctx, uint32_t first_task, uint32_t n, const uint32_t* class_id, const uint64_t* priority);
/* Declares priority values before any task carries them.  Needed when the ready set is sharded over
 * several contexts (every rank must number the priority levels identically).  A context whose levels were declared
 * does not prune them on its own (the ranks would diverge): the caller prunes them over all ranks with
 * hqs_levels_live and hqs_levels_retain, between ticks. */
int hqs_levels_add(hqs_ctx* ctx, uint32_t n, const uint64_t* priority);
/* The context's exact level table (registered priorities, descending) and, per level, whether a VALID key of this
 * context carries it (1) or not (0).  *n_levels (optional) receives the table size; with cap == 0 nothing else is done,
 * otherwise cap must be >= the table size.  A level dead on this rank may be live on another: the ranks OR their live
 * vectors before hqs_levels_retain.  HQS_E_STATE while a tick has not been fetched. */
int hqs_levels_live(hqs_ctx* ctx, uint32_t cap, uint64_t* levels, uint8_t* live, uint32_t* n_levels);
/* Keeps the levels with keep[i] != 0 (i indexes the table hqs_levels_live returned), drops the others, rebuilds the
 * device table and re-keys every VALID task.  HQS_E_INVALID, with nothing changed, if n is not the table size or a
 * dropped level is still carried by a VALID key of this context.  Every rank must pass the same keep vector. */
int hqs_levels_retain(hqs_ctx* ctx, uint32_t n, const uint8_t* keep);
/* TaskQueue::remove (taskqueue.rs:194-216): cancel / externally assigned tasks leave the ready set.  Also the way to
 * retire the handle of a task that has FINISHED: a removed handle leaves the device table, so it no longer pins its
 * priority level (levels without any task are pruned when the level set outgrows HQS_MAX_GROUPS / n_classes or doubles;
 * tako priorities carry a per-job component, so a long-running server would otherwise accumulate one level per job). */
int hqs_ready_remove(hqs_ctx* ctx, uint32_t n, const uint32_t* task);

/* DAG mode (reactor.rs:188-220 on_new_tasks + :500-580 task_finished, device resident): loads a whole
 * task graph; tasks with n_deps == 0 are ready at once.  consumers of task t are
 * cons[cons_off[t] .. cons_off[t+1]).  Handles are 0..n_tasks-1 and replace the current table. */
int hqs_dag_load(hqs_ctx* ctx, uint32_t n_tasks, const uint32_t* class_id, const uint64_t* priority,
                 const uint32_t* n_deps, const uint32_t* cons_off, const uint32_t* cons);
/* task_finished for n tasks: decrements unfinished_deps of every consumer; consumers reaching zero
 * become ready (add_ready_task).  *n_new_ready (optional) receives how many did.  A handle >= n_tasks rejects the batch
 * (HQS_E_INVALID, nothing changed). */
int hqs_tasks_finished(hqs_ctx* ctx, uint32_t n, const uint32_t* task, uint32_t* n_new_ready);

/* Task graphs that grow while the ready set runs (reactor.rs:188-220 on_new_tasks, :500-580 task_finished): jobs with
 * dependencies are submitted between ticks into the same table that hqs_ready_push fills.
 * hqs_graph_push: on_new_tasks for n NEW tasks with dependencies.  task[i], class_id[i], priority[i] as in hqs_ready_push
 * (priorities are registered the same way); the dependencies of task i are deps[dep_off[i] .. dep_off[i+1]) (handles).
 * A dependency counts if its handle is VALID (waiting, ready, or assigned and not finished) or is an EARLIER task of the
 * batch; one on a later task of the batch, or on a handle that finished, was removed or never pushed, is dropped, as
 * on_new_tasks drops a dependency it does not find.  A task without a counted dependency is READY at once, the others wait
 * (VALID, neither READY nor DONE).  *n_ready (optional) = how many of the n tasks are ready at once.
 * HQS_E_INVALID with nothing changed: a class id >= n_classes; a handle 0xFFFFFFFF, a handle twice in the batch, or a
 * handle that is VALID; a task that depends on itself or names a dependency twice; a dependency that is neither in the
 * batch nor < n_handles; dep_off not starting at 0 or decreasing.
 * hqs_graph_finished: task_finished for n tasks: each leaves the table (like hqs_ready_remove), and then each consumer still
 * waiting on the incarnation it was submitted with loses a dependency; the ones reaching zero become READY.  *new_ready
 * points to their handles, ASCENDING, in a buffer the context owns, valid until the next call on the context;
 * *n_new_ready is their number.  A handle >= n_handles rejects the batch (HQS_E_INVALID, nothing changed); a handle that
 * is not VALID is ignored (tako's "unknown task finished"); a handle named twice counts once.  A consumer finished in the
 * same batch is not released.
 * Handle re-use: a task that leaves the table (hqs_graph_finished, hqs_ready_remove or hqs_graph_cancel) takes its consumer
 * list with it.  The consumers of a task removed with hqs_ready_remove keep waiting until the host removes them too;
 * hqs_graph_cancel removes a task together with its consumers.  A handle that is submitted again is a new incarnation: the
 * producers of the old one never release it.
 * hqs_graph_cancel: on_cancel_tasks / task_failed (reactor.rs:596-770) for n tasks.  Every named handle that is VALID
 * (waiting, ready, prefilled or assigned) leaves the table, and so does, transitively, every consumer still waiting on the
 * incarnation its edge was made for (a consumer cancelled or resubmitted since is not followed).  Leaving is what
 * hqs_graph_finished does to a task (READY, VALID, DONE and PREFILLED cleared, so it stops pinning its priority level)
 * without releasing anyone; the consumer lists of all of them are emptied.  *cancelled points to every handle that left,
 * ASCENDING (the named VALID ones and the consumers reached), in the buffer hqs_graph_finished uses, valid until the next
 * call on the context; *n_cancelled is their number.  The consumers are that list without the named handles.  A handle
 * that is not VALID is ignored, a handle named twice counts once.  HQS_E_INVALID with nothing changed: a handle >=
 * n_handles, or task == NULL with n > 0.  The number of kernel launches does not depend on the depth of the graph (one
 * cooperative kernel marks the whole closure); a marking that makes no progress for about a second fails with
 * HQS_E_CUDA and changes nothing.
 * hqs_ready_push / _range / _remove / _rearm, prefill, ticks, queries and the grouped fetch work unchanged on a graph
 * context.  HQS_E_STATE: the graph calls after hqs_dag_load, on a context attached with hqs_shard_attach or set up with
 * hqs_shard_graph_init, or while a tick or query is pending; hqs_dag_load after a graph push.
 * hqs_graph_debug (debug / test aid, like hqs_debug_keys): out[0] live edges (linked into a producer's consumer list),
 * out[1] edge-pool capacity, out[2] pool compactions so far, out[3] waiting tasks (VALID, not READY, not DONE). */
int hqs_graph_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id, const uint64_t* priority,
                   const uint32_t* dep_off, const uint32_t* deps, uint32_t* n_ready);
int hqs_graph_finished(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** new_ready, uint32_t* n_new_ready);
int hqs_graph_cancel(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** cancelled, uint32_t* n_cancelled);
int hqs_graph_debug(hqs_ctx* ctx, uint64_t out[4]);

/* Retires the handles of forgotten tasks: an order-preserving renumbering of the task table, so that a long-running server's
 * tick cost and memory follow its live tasks, not every task it has ever seen.
 * Survivors: every handle whose key is VALID (waiting, ready, prefilled, or assigned and not finished or removed), plus the
 * handles named in keep[0 .. n_keep).  keep may name handles in any state, in any order, and more than once; the host names
 * there the tasks it still tracks that have left the table (for example a prefilled task a worker started, which
 * hqs_ready_remove took out).
 * Renumbering: survivor i, in ascending old handle, becomes handle i, so handle order stays TaskId order and new handles
 * keep being appended after the survivors.  *old_of_new points to the *n_kept old handles, ascending, in the buffer
 * hqs_graph_finished uses, valid until the next call on the context.  n_handles (and hqs_stats.n_handles) becomes n_kept.
 * What moves with a survivor: its key verbatim (READY, DONE, VALID and PREFILLED bits, level and class), its priority and,
 * on a graph context, its dependency count, its incarnation and its consumer list, with the consumers renumbered.  An edge
 * whose consumer no longer waits on the edge's incarnation is dropped, as a pool compaction drops it.
 * The slots [n_kept, old n_handles) become slots that were never used: key 0, no dependencies, incarnation 0, an empty
 * consumer list.  Capacity is kept.  The level table, the class table, the prefill configuration and the prefill mask given
 * with hqs_prefill_state are unchanged.
 * HQS_E_INVALID with nothing changed: a keep entry >= n_handles, or keep == NULL with n_keep > 0.  HQS_E_STATE with nothing
 * changed: a tick or query is pending, after hqs_dag_load, on a context attached with hqs_shard_attach or set up with
 * hqs_shard_graph_init.  A failed allocation or CUDA error (HQS_E_CUDA) leaves the context as it was: the survivors are
 * gathered into fresh arrays that replace the table only at the end.
 * The number of kernel launches does not depend on n_handles (at most eight); the call synchronises with the host twice
 * (the survivor count, then the copy of *old_of_new) and does no per-handle work on the host. */
int hqs_handles_compact(hqs_ctx* ctx, uint32_t n_keep, const uint32_t* keep, const uint32_t** old_of_new, uint32_t* n_kept);

/* Task graphs over a sharded ready set: the graph is replicated on every rank, each task's key lives on its owner.
 * hqs_shard_graph_init: this context owns the GLOBAL handles [lo, hi) of a graph over n_total handles (its key table holds
 * handle h at h - lo, as in the sharded tick) and allocates the replicated graph (the three per-handle arrays and the work
 * list of hqs_graph_cancel, one VALID bit per handle, over all n_total handles, and the edge pool).  Allowed on attached
 * contexts and on the contexts of the NCCL form.  HQS_E_STATE after hqs_dag_load or a hqs_graph_push, when the table holds a
 * VALID key, a second time, or while a tick or query is pending; HQS_E_INVALID for lo > hi or hi > n_total.  From then on
 * every task enters through hqs_shard_graph_push (a task without dependencies too), every remove goes through
 * hqs_shard_graph_remove: hqs_ready_push, hqs_ready_push_range, hqs_ready_remove and the single-context graph calls return
 * HQS_E_STATE, and the calls below return it on any other context.
 * Every rank makes every call below with the same arguments (GLOBAL handles) and runs the same propagation on the same
 * replicated state; no data moves between ranks.  A rank writes only the keys it owns and reports only the handles it owns,
 * so the concatenation of the ranks' outputs in rank order is what one context holding every task returns.
 * hqs_shard_graph_push: hqs_graph_push for the whole batch, with its contract and rejections; the bound for handles and
 * dependencies is n_total (a handle or a dependency >= n_total rejects the batch on every rank).  Every priority of the batch
 * must have been declared with hqs_levels_add (on every rank), and a class id >= n_classes is found on the host, so every rank
 * rejects the same batches.  *n_ready counts this rank's tasks that are ready at once.
 * hqs_shard_graph_finished: hqs_graph_finished; *new_ready = the newly ready handles this rank owns, global, ascending.
 * hqs_shard_graph_cancel: hqs_graph_cancel; every rank marks the whole closure and removes it from its replica, and
 * *cancelled = the part of the closure this rank owns, global, ascending.  The same six launches at any depth.
 * hqs_shard_graph_remove: hqs_ready_remove for global handles: the owner's keys leave the table, every rank empties the
 * handles' consumer lists and clears their graph VALID bits.  A handle >= n_total rejects the batch (HQS_E_INVALID).
 * hqs_graph_debug answers on a sharded graph context: out[0..2] describe the replicated graph (equal on every rank), out[3]
 * counts this rank's own waiting tasks.
 * Every rejection (HQS_E_INVALID, HQS_E_STATE, HQS_E_LIMIT) follows from the arguments and the replicated state, so every rank
 * rejects alike and nothing changes.  HQS_E_CUDA from any of these calls (a CUDA error, a failed allocation, the cancel
 * marking's time-out) happens on one rank only and may leave that rank's replica different from the others: the context
 * then refuses every sharded graph call with HQS_E_STATE, and the server must tear the sharded graph down on every rank. */
int hqs_shard_graph_init(hqs_ctx* ctx, uint32_t n_total, uint32_t lo, uint32_t hi);
int hqs_shard_graph_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id, const uint64_t* priority,
                         const uint32_t* dep_off, const uint32_t* deps, uint32_t* n_ready);
int hqs_shard_graph_finished(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** new_ready, uint32_t* n_new_ready);
int hqs_shard_graph_cancel(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** cancelled, uint32_t* n_cancelled);
int hqs_shard_graph_remove(hqs_ctx* ctx, uint32_t n, const uint32_t* task);

/* hqs_handles_compact over a sharded graph: every rank renumbers the replicated graph alike and keeps its own tasks.  It reads
 * like hqs_handles_compact, with global handles, and no key moves between ranks.
 * Survivors: every global handle whose replicated graph VALID bit is set, plus the GLOBAL handles named in keep[0 .. n_keep)
 * (any order, repeats allowed).  The survivor set is computed from replicated state only, so every rank must pass the same
 * keep list (ShardedScheduler.compact_handles gathers what each rank tracks).
 * Renumbering: survivor i, in ascending old handle, becomes global handle i.  *old_of_new points to the *n_kept old handles,
 * ascending, the same list on every rank, in the buffer hqs_graph_finished uses, valid until the next call on the context.
 * New ranges: with new(h) = the number of survivors below h, and new(n_total) = n_total, a rank that owned [lo, hi) now owns
 * [new(lo), new(hi)), written to new_range[0..1] (which may be NULL).  So the rank whose range ends at n_total (the last rank)
 * owns [new(lo), n_total), the freed tail [n_kept, n_total) included, the ranges still tile [0, n_total) in rank order (the
 * order the global rank inside a group depends on), and every survivor's key stays on the rank that owns it.  n_total is
 * unchanged; new tasks, numbered after the survivors, land on the last rank.
 * What moves with a survivor on every rank: its graph VALID bit, dependency count, incarnation and consumer list, with the
 * consumers renumbered; an edge whose consumer no longer waits on the edge's incarnation is dropped.  On its owner only: its
 * key verbatim (READY, DONE, VALID and PREFILLED bits, level and class) and its priority, now at new(h) - new(lo).  The rank's
 * n_handles (and hqs_stats.n_handles) becomes its own survivor count (the last rank counts up to n_kept, not n_total).
 * Unchanged: the level table, the class table, the prefill configuration and mask, the exchange buffers and the peer-to-peer
 * sequence state.  The key table's capacity is kept (or grown to the own survivor count), and the last rank's table grows into
 * the tail as pushes reach it.
 * Rejections leave every rank unchanged and happen alike on every rank: HQS_E_INVALID for a keep entry >= n_total or
 * keep == NULL with n_keep > 0; HQS_E_STATE where the sharded graph calls refuse (no hqs_shard_graph_init, which includes a
 * sharded ready set without a graph, a replica marked failed, a pending tick or query).  HQS_E_CUDA marks the replica failed
 * like every other sharded graph call; the rank's own arrays stay as they were (fresh arrays are swapped in only at the end).
 * hqs_handles_compact still returns HQS_E_STATE on a sharded graph context.
 * At most nine kernel launches whatever n_total is; the call synchronises with the host twice (the survivor count and the
 * new ranges, then the copy of *old_of_new). */
int hqs_shard_graph_compact(hqs_ctx* ctx, uint32_t n_keep, const uint32_t* keep, const uint32_t** old_of_new,
                            uint32_t* n_kept, uint32_t new_range[2]);

/* One scheduler tick over the current ready set (replaces run_scheduling_solver + the task-selection
 * half of create_task_mapping).
 *   workers[n_workers]            ascending worker_id
 *   free_rw[n_workers][R]         SingleNodeTaskAssignment::free_resources   (worker.rs:44)
 *   total_rw[n_workers][R]        Worker::resources                          (worker.rs:69)
 *   blocked_wcv                   optional bitmask, bit index ((w * n_classes + c) * HQS_MAX_VARIANTS + v),
 *                                 LSB-first in bytes: Worker::blocked_requests (worker.rs:70,328-344)
 *   out[out_cap], *out_n          assignments (kind 0 / 2), ordered by (priority desc, class order of this tick,
 *                                 handle asc), then the prefill records (kind 1) if proactive filling is on — per worker that is already the priority-descending
 *                                 order mapping.rs:125-128 sorts into
 *   free_after[n_workers][R]      optional: free vectors after the tick's assignments
 * Assigned tasks leave the ready set (Waiting -> Assigned, mapping.rs:55-66). */
int hqs_tick(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
             const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t out_cap,
             hqs_assignment* out, uint32_t* out_n, uint64_t* free_after);

/* Split form of hqs_tick for pipelining / device-side timing: launch enqueues the upload of the worker
 * state and the tick kernels on the context stream and returns; fetch waits and copies the result.
 * hqs_tick(...) == hqs_tick_launch(...) followed by hqs_tick_fetch(...). */
int hqs_tick_launch(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers,
                    const uint64_t* free_rw, const uint64_t* total_rw, const uint8_t* blocked_wcv,
                    uint32_t out_cap);
int hqs_tick_fetch(hqs_ctx* ctx, uint32_t out_cap, hqs_assignment* out, uint32_t* out_n,
                   uint64_t* free_after);

/* hqs_tick_fetch with the records regrouped by worker on the device, the shape tako sends them in (one message list per
 * worker, WorkerTaskMapping::send_messages, mapping.rs:255-288).  With W = n_workers of the launch and n = *out_n:
 *   out[ worker_off[2w]   .. worker_off[2w+1] )   worker w's prefill records (kind 1), in emission order
 *   out[ worker_off[2w+1] .. worker_off[2w+2] )   worker w's assignments (kind 0), in emission order = priority descending
 *   out[ worker_off[2W]   .. worker_off[2W+1] )   all redirect records (kind 2), in emission order, NOT grouped: the
 *                                                 RetractTasks message goes to the worker the task was prefilled on, which
 *                                                 only the host knows
 *   worker_off[0] = 0, worker_off[2W+1] = n, non-decreasing, 2W + 2 entries
 * i.e. a stable sort of what hqs_tick_fetch returns by key = kind == 2 ? 2W : 2 * worker + (kind == 0); the records keep
 * their 8-byte form.  It fetches whatever tick is pending (hqs_tick_launch, hqs_shard_tick_launch, hqs_shard_solve_emit: a
 * rank gets its own records grouped).  States and errors are hqs_tick_fetch's; in addition a null worker_off or
 * off_cap < 2W + 2 returns HQS_E_INVALID and leaves the tick fetchable by either fetch.  The grouping kernels run at fetch
 * time, so a failed tick launches nothing, and n == 0 launches nothing and returns an all-zero table.
 *   hqs_tick_grouped     = hqs_tick_launch + hqs_tick_fetch_grouped
 *   hqs_grouped_reserve  allocates what the grouped fetch needs for n_workers and out_cap records and loads its kernels
 *                        (otherwise done by the first grouped fetch); contexts that wait for each other on the device call
 *                        it before their first tick, as hqs_tick_reserve.  A context that never fetches grouped never pays.
 *   hqs_grouped_kernel_ms  device time of the grouping kernels of the last grouped fetch, between two CUDA events on the
 *                        context stream (hqs_set_profile on; HQS_E_STATE if there is none). */
int hqs_tick_fetch_grouped(hqs_ctx* ctx, uint32_t out_cap, hqs_assignment* out, uint32_t* out_n, uint32_t off_cap,
                           uint32_t* worker_off, uint64_t* free_after);
int hqs_tick_grouped(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                     const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t out_cap, hqs_assignment* out,
                     uint32_t* out_n, uint32_t off_cap, uint32_t* worker_off, uint64_t* free_after);
int hqs_grouped_reserve(hqs_ctx* ctx, uint32_t n_workers, uint32_t out_cap);
int hqs_grouped_kernel_ms(hqs_ctx* ctx, float* out_ms);

/* What-if query (scheduler/query.rs:12-131, ServerRef::new_worker_query control.rs:123-136): runs the histogram
 * and the solver against an arbitrary (e.g. hypothetical, autoalloc) worker array WITHOUT emitting or consuming
 * anything: the ready set is unchanged.  per_worker_assigned[n_workers] (optional) receives how many tasks each
 * worker would get — a fake worker is "needed" iff its count is > 0; free_after as in hqs_tick.  Partial
 * descriptors use HQS_AMOUNT_MAX for unknown resources (query.rs:35-46).
 * On a context of a sharded ready set (hqs_shard_attach) hqs_query answers for the tasks of THIS rank only; the answer over
 * all ranks is hqs_shard_query_launch (or hqs_shard_count + hqs_shard_query_solve) on every rank, below. */
int hqs_query(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
              const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t* n_would_assign,
              uint32_t* per_worker_assigned, uint64_t* free_after);
/* Fetches a query launched by hqs_shard_query_launch or hqs_shard_query_solve (hqs_query == launch + this fetch on one
 * context): outputs as in hqs_query, with the launch's n_workers entries.  A query is pending like a tick until it is
 * fetched: every call that fails with "the previous tick has not been fetched" fails the same way, hqs_tick_fetch on a
 * pending query and hqs_query_fetch on a pending tick or with nothing pending return HQS_E_STATE and leave the pending launch
 * fetchable.  A query does not count in hqs_stats.ticks. */
int hqs_query_fetch(hqs_ctx* ctx, uint32_t* n_would_assign, uint32_t* per_worker_assigned, uint64_t* free_after);

/* Multi-GPU sharding (SURVEY.md §8(e)): each rank owns a contiguous handle range of the task table.
 * Phase 1 counts the rank's ready tasks per group into d_counts (device pointer, n_groups_cap u32).
 * The host all-gathers the count vectors (NCCL), then phase 2 runs the replicated deterministic solve
 * on the summed counts and emits only this rank's tasks; ranks_before = element-wise sum of the count
 * vectors of lower ranks, counts_all = sum over all ranks (device pointers). */
int hqs_shard_count(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers,
                    const uint64_t* free_rw, const uint64_t* total_rw, const uint8_t* blocked_wcv,
                    uint32_t* d_counts, uint32_t n_groups_cap, uint32_t* n_groups);
int hqs_shard_solve_emit(hqs_ctx* ctx, const uint32_t* d_counts_all, const uint32_t* d_ranks_before,
                         uint32_t out_cap);
/* Allocates every buffer a tick over n_workers workers and up to out_cap assignments needs (they are otherwise
 * allocated by the first tick).  cudaMalloc synchronises the device, so contexts that wait for each other on the
 * device (the peer exchange below, several contexts of one process) reserve before their first tick. */
int hqs_tick_reserve(hqs_ctx* ctx, uint32_t n_workers, uint32_t out_cap, int with_blocked);

/* Sharded tick WITHOUT a host collective: the count vectors travel by peer-to-peer stores (NVLink) straight from
 * the counting step into every rank's exchange buffer and the solver kernel waits for them on the device.
 *   hqs_shard_xbuf     allocates this context's exchange buffer; returns its device pointer and its CUDA IPC handle
 *   hqs_ipc_open       maps another process's exchange buffer (handle from its hqs_shard_xbuf) into this process
 *   hqs_shard_attach   peer_xbufs[r] = exchange buffer of rank r as seen from this process (own buffer at [rank];
 *                      contexts of one process pass each other's pointers directly)
 *   hqs_shard_tick_launch = hqs_tick_launch for rank `rank` of `world`: count -> peer stores + release flag ->
 *                      solve (acquires all flags, sums the vectors; same deterministic solve on every rank) ->
 *                      emit of this rank's tasks.  Fetch with hqs_tick_fetch.  All ranks must tick in lockstep.
 * Every rank publishes its number G of (level, class) groups next to its flag.  If a peer's G differs (for example proactive
 * filling on one rank and off on another), hqs_tick_fetch returns HQS_E_STATE on every rank, with a text naming both counts;
 * nothing was solved or emitted and the ready sets are unchanged.  Only G is compared: ranks with the same G but different
 * prefill reserve / max values, or different level or class sets with the same number of groups, are NOT detected and
 * silently compute different results; keeping them identical is the caller's job. */
#define HQS_IPC_HANDLE_BYTES 64
int hqs_shard_xbuf(hqs_ctx* ctx, void** d_xbuf, uint8_t ipc_handle[HQS_IPC_HANDLE_BYTES]);
int hqs_ipc_open(hqs_ctx* ctx, const uint8_t ipc_handle[HQS_IPC_HANDLE_BYTES], void** d_ptr);
int hqs_shard_attach(hqs_ctx* ctx, uint32_t world, uint32_t rank, void* const* peer_xbufs);
int hqs_shard_tick_launch(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                          const uint64_t* total_rw, const uint8_t* blocked_wcv, uint32_t out_cap);

/* What-if query over a sharded ready set.  Contract: every rank holds the same classes, declared levels, prefill
 * configuration and fake-worker array; then every rank returns the same answer, and it is what hqs_query returns on ONE
 * context holding the union of the ranks' ready sets (n_would_assign, per-worker counts, free vectors, bit for bit).  Nothing
 * is emitted or consumed on any rank.  Fetch with hqs_query_fetch on every rank.
 *   hqs_shard_query_launch  fused form, the counterpart of hqs_shard_tick_launch: one tick kernel with the peer exchange and
 *                           without the emit step.  Ticks and queries share one exchange sequence, so all ranks must call it
 *                           in lockstep, like a tick.  After hqs_tick_reserve with at least n_workers it allocates nothing
 *                           (contexts of one process wait for each other on the device).  Ranks with different G fail it as a
 *                           tick: hqs_query_fetch returns HQS_E_STATE on every rank, naming both counts; the ready sets are
 *                           unchanged.
 *   hqs_shard_query_solve   NCCL form: after hqs_shard_count (same worker array) with the all-gathered totals counts_all
 *                           (device pointer, as for hqs_shard_solve_emit; a query emits nothing, so no ranks_before). */
int hqs_shard_query_launch(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                           const uint64_t* total_rw, const uint8_t* blocked_wcv);
int hqs_shard_query_solve(hqs_ctx* ctx, const uint32_t* d_counts_all);
/* Device pointer / length of the last tick's assignment buffer (for NCCL all-gather of results).  *d_out_n counts the
 * assignments (kind 0 / 2) only; with proactive filling on, the tick's prefill records (kind 1) follow them in d_out and
 * hqs_tick_fetch's *out_n counts both. */
int hqs_device_result(hqs_ctx* ctx, const hqs_assignment** d_out, const uint32_t** d_out_n);

/* Proactive filling (scheduler/mapping.rs:156-230, SchedulerConfig::proactive_filling_reserve / _max, state.rs:14-21;
 * tako's defaults are 16 / 40).  Off (max = 0) unless configured.  With it on, a tick
 *   - counts prefilled tasks as ready; inside one priority level the waiting tasks of a class go first, the prefilled
 *     ones second (TaskQueue::take_tasks, taskqueue.rs:320-355); an assigned prefilled task comes out with kind = 2,
 *   - appends, behind the assignments, kind = 1 records: for every class whose best level with waiting tasks is the best
 *     over all classes, the workers that received an assignment of the class in this tick and hold no prefilled task of
 *     it (hqs_prefill_state) each get min((waiting tasks of the level - reserve) / workers, max) of the next waiting tasks.
 * The host keeps Worker::prefilled_tasks: it passes "worker w holds a prefilled task of class c" before each tick
 * (hqs_prefill_state, bytes [n_workers][n_classes], consumed by the next tick), removes a prefilled task that a worker
 * started with hqs_ready_remove, and calls hqs_prefill_dispose(class) where TaskQueue::check_dispose_prefill
 * (taskqueue.rs:146-152: a task of higher priority became ready) retracts the class's prefills.
 * Sharded ticks (hqs_shard_count + hqs_shard_solve_emit, hqs_shard_tick_launch): every rank is configured with the same
 * hqs_prefill_config and is given the same GLOBAL mask before each tick (worker w holds a prefilled task of class c, over
 * the tasks of all ranks: only the host knows it).  The solve is replicated, so every rank computes the same prefill
 * ranges; each rank emits the kind-1 records of its own tasks, behind its own assignments and in single-context order, and
 * marks only those tasks prefilled.  hqs_prefill_dispose(class) is called on every rank and clears the rank's own tasks. */
int hqs_prefill_config(hqs_ctx* ctx, uint32_t reserve, uint32_t max_per_worker);
int hqs_prefill_state(hqs_ctx* ctx, uint32_t n_workers, const uint8_t* prefilled_wc);
int hqs_prefill_dispose(hqs_ctx* ctx, uint32_t class_id);

/* Restores every task that earlier ticks assigned (DONE) to the ready state (benchmark and what-if use:
 * re-arm the same ready set without a new upload). */
int hqs_ready_rearm(hqs_ctx* ctx);

void* hqs_stream(hqs_ctx* ctx);                 /* cudaStream_t of the context                */
/* Makes the context enqueue its work on an externally owned stream (e.g. the host framework's current
 * stream) so that several contexts serialise on one stream and foreign events can time them. */
int hqs_set_stream(hqs_ctx* ctx, void* cuda_stream);
/* Device timing of the tick (off by default).  out_ms[3] = the tick kernel between two CUDA events on the context
 * stream; out_ms[0..2] = its phases as seen by the solver CTA's clock (staging + wait for the histogram, exchange +
 * compaction + solve, emit), scaled to out_ms[3].  Valid after the tick has been fetched. */
int hqs_set_profile(hqs_ctx* ctx, int on);
int hqs_get_kernel_ms(hqs_ctx* ctx, float out_ms[4]);
/* Debug: phase lengths of the solver CTA of the last fetched tick in SM clock cycles: [0] staging + wait for the
 * histogram, [1] exchange + compaction + demand, [2] the solver warp, [3] emit, [4] non-empty groups, [5] whole
 * kernel, [6] whole kernel in nanoseconds (globaltimer), [7] pack commands. */
int hqs_debug_read(hqs_ctx* ctx, uint64_t out[8]);
/* Debug / test aid: waits for the context stream and copies the first min(cap, n_handles) words of the device task table
 * (key[h]: bit31 READY, bit30 DONE, bit29 VALID, bit28 PREFILLED, bits 14..27 the priority level, bits 0..13 the class)
 * into keys; *n_handles (optional) receives the table size.  HQS_E_STATE while a tick has not been fetched. */
int hqs_debug_keys(hqs_ctx* ctx, uint32_t cap, uint32_t* keys, uint32_t* n_handles);
int hqs_sync(hqs_ctx* ctx);
int hqs_get_stats(hqs_ctx* ctx, hqs_stats* out);

#ifdef __cplusplus
}
#endif
#endif /* HQSCHED_H */
