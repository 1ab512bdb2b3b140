// tako_shim.hpp — C++ host side of the scheduler tick above the C ABI of hqsched.h.
//
// The reference's host code for this path is Rust (crates/tako/src/internal/scheduler, .../server).  No Rust
// toolchain exists in the build image, so the shim a tako maintainer would write in Rust (INTEGRATION.md) is
// written here in C++ with the reference's names, argument meaning and error behaviour:
//
//   reference (Rust, file:line)                                       here
//   ----------------------------------------------------------------  -------------------------------------
//   ResourceAllocRequest / ResourceRequest / ResourceRequestVariants  same names        request.rs:13-83,136-353
//   ResourceRqMap::get_or_create (map.rs:99-109, control.rs:222-227)  GpuCore::get_or_create_resource_rq_id
//   Priority::from_user_priority (priority.rs:43-48)                  priority_from_user
//   on_new_worker / on_remove_worker (reactor.rs:20-32, 64-186)       GpuCore::on_new_worker / on_remove_worker
//   Worker::block_request / unblock (worker.rs:328-344)               GpuCore::block_request / unblock_request
//   on_new_tasks (reactor.rs:188-220)                                 GpuCore::on_new_tasks (handles in TaskId order)
//   on_new_tasks with dependencies (reactor.rs:188-220)               GpuCore::on_new_tasks(std::vector<NewTask>)
//   TaskQueues::add_ready_task (taskqueue.rs:37-43)                   GpuCore::add_ready_task
//   TaskQueue::remove (taskqueue.rs:194-216)                          GpuCore::remove_ready_task
//   run_scheduling_inner (main.rs:40-46) -> WorkerTaskMapping         GpuCore::run_scheduling
//   WorkerTaskMapping / WorkerTaskUpdate (mapping.rs:9-21)            same names
//   task_finished -> Worker::remove_sn_task (reactor.rs:500-580,      GpuCore::on_task_finished
//                    workerload.rs:194-202)
//   on_cancel_tasks (reactor.rs:696-770)                              GpuCore::on_cancel_tasks
//   task_failed (reactor.rs:596-694)                                  GpuCore::on_task_failed
//
// Error behaviour follows the reference: the scheduler never returns errors to its caller.  A failing tick logs
// the library's message and schedules nothing (solver.rs:412-415); invalid requests ("Zero resources cannot be
// requested", request.rs:24-32) are programming errors and throw std::invalid_argument, the analogue of the
// reference's panics.
#pragma once

#include <cstdint>
#include <map>
#include <optional>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "hqsched.h"

namespace tako_b200 {

using ResourceId = uint32_t;
using ResourceAmount = uint64_t;          // fixed point, 10 000 fractions per unit (amount.rs:7)
using ResourceRqId = uint32_t;
using ResourceVariantId = uint8_t;
using WorkerId = uint32_t;
using Priority = uint64_t;
constexpr ResourceAmount FRACTIONS_PER_UNIT = 10000;

struct TaskId {                           // ids.rs:17-21: ordered by (job_id, job_task_id)
    uint32_t job_id = 0, job_task_id = 0;
    uint64_t as_u64() const { return ((uint64_t)job_id << 32) | job_task_id; }
    bool operator==(const TaskId& o) const { return as_u64() == o.as_u64(); }
    bool operator<(const TaskId& o) const { return as_u64() < o.as_u64(); }
};

inline Priority priority_from_user(int32_t user_priority) {
    return (uint64_t)((uint32_t)user_priority ^ 0x80000000u) << 32;
}

struct ResourceAllocRequest {             // request.rs:50-83; the five amount policies are one case server-side
    ResourceId resource_id = 0;
    bool all = false;                     // AllocationRequest::All
    ResourceAmount amount = 0;
};
struct ResourceRequest {                  // request.rs:136-227
    std::vector<ResourceAllocRequest> entries;
    uint64_t min_time_ms = 0;
    uint32_t weight = 10000;              // ResourceWeight raw value
    uint32_t n_nodes = 0;
};
struct ResourceRequestVariants {          // request.rs:229-353
    std::vector<ResourceRequest> variants;
};

struct NewTask {                          // a submitted task with its dependencies (task.rs:22-43, reactor.rs:188-220)
    TaskId id;
    ResourceRqId rq = 0;
    Priority priority = 0;
    std::vector<TaskId> deps;
};

struct WorkerTaskUpdate {                 // mapping.rs:9-14
    std::vector<std::pair<TaskId, ResourceVariantId>> assigned;   // priority descending (mapping.rs:125-128)
    std::vector<TaskId> prefills;         // ComputeTasks entries with variant = None, sent BEFORE the assigned ones (mapping.rs:264-275)
    std::vector<TaskId> retracts;         // one RetractTasks message, sent first (mapping.rs:257-262)
};
struct CancelledTasks {                   // on_cancel_tasks (reactor.rs:696-770)
    std::vector<TaskId> cancelled;        // every task that left, the named ones and their consumers, ascending TaskId
    std::map<WorkerId, std::vector<TaskId>> messages;   // CancelTasks per worker, tasks in the order they were named
};
struct WorkerTaskMapping {                // mapping.rs:16-21
    std::map<WorkerId, WorkerTaskUpdate> workers;
    size_t n_assigned() const {
        size_t n = 0;
        for (const auto& kv : workers) n += kv.second.assigned.size();
        return n;
    }
};

// The slice of Core + SchedulerState the tick needs (core.rs:22-110, scheduler/state.rs:23-28), with the ready
// set resident on the GPU.
class GpuCore {
public:
    explicit GpuCore(uint32_t n_resources, int device = 0, uint32_t create_flags = 0);
    ~GpuCore();
    GpuCore(const GpuCore&) = delete;
    GpuCore& operator=(const GpuCore&) = delete;

    ResourceRqId get_or_create_resource_rq_id(const ResourceRequestVariants& rqv);

    // resources[r] = total of resource r (missing => 0); termination_ms: absolute time in ms, nullopt = none
    void on_new_worker(WorkerId id, const std::vector<ResourceAmount>& resources, float min_utilization = 0.0f,
                       std::optional<uint64_t> termination_ms = std::nullopt);
    // running tasks of the worker become ready again (reactor.rs:104-150)
    void on_remove_worker(WorkerId id);
    void block_request(WorkerId id, ResourceRqId rq, ResourceVariantId v);
    void unblock_request(WorkerId id, ResourceRqId rq, ResourceVariantId v);

    // on_new_tasks (reactor.rs:188-220): announces the tasks of a submit; handles are assigned in ascending TaskId
    void on_new_tasks(std::vector<TaskId> tasks);
    // on_new_tasks for tasks with dependencies: handles are assigned in TaskId order; a dependency on an unknown, finished
    // or cancelled task is dropped (reactor.rs:197-204), one on a live task (waiting, ready, assigned or running) counts.
    // Tasks without a counted dependency become ready; the others wait until their producers finish.  The tasks go to the
    // device in one hqs_graph_push at the next flush, and from then on this core's finished tasks release their consumers
    // through hqs_graph_finished.
    void on_new_tasks(std::vector<NewTask> tasks);
    size_t n_waiting() const;             // tasks waiting for a dependency
    void add_ready_task(TaskId task, ResourceRqId rq, Priority priority);
    void remove_ready_task(TaskId task);

    WorkerTaskMapping run_scheduling(uint64_t now_ms = 0);
    // The same tick and the same WorkerTaskMapping, list order included, with the records regrouped per worker on the
    // device (hqs_tick_grouped): one map lookup and one reserved append per worker and section instead of a lookup and a
    // push_back per record.  Defined in tako_shim_grouped.cpp.
    WorkerTaskMapping run_scheduling_grouped(uint64_t now_ms = 0);
    void on_task_finished(TaskId task);
    // on_cancel_tasks (reactor.rs:696-770): the named tasks that are known and not finished leave, and so do, transitively,
    // all their waiting consumers (hqs_graph_cancel; a core that never submitted dependencies has none).  An assigned or
    // running task gives its resources back and is cancelled on its worker, a prefilled one on the worker holding it, a
    // retracting one on the worker it is being retracted from (its redirect is dropped and the target's resources come
    // back).  Pending submits and finishes are flushed first.  Defined in tako_shim_graph_cancel.cpp.
    CancelledTasks on_cancel_tasks(const std::vector<TaskId>& tasks);
    // task_failed (reactor.rs:596-694): the failing task leaves as a cancelled one does, without a message to its worker;
    // returns its transitive consumers, ascending TaskId (the list tako hands to on_task_error), which left with it.
    std::vector<TaskId> on_task_failed(TaskId task);

    // Retires the handles of the tasks tako has forgotten (finished, or cancelled or failed with their consumers): pending
    // submits and finishes are flushed, the device table is renumbered in TaskId order without them (hqs_handles_compact) and
    // the host mirror with it.  Every other task keeps a handle, whatever its state.  Returns the number of handles retired.
    // The embedding server decides when, for example when n_handles() exceeds twice the tasks it knows.  Defined in
    // tako_shim_retire.cpp.
    size_t retire_handles();
    size_t n_handles() const { return tasks_.size(); }   // handles given out and not retired
    // Test aid: handle_of throws std::length_error once `end` handles are in use (default: the whole 32-bit space, less
    // 0xFFFFFFFF, which the C ABI reserves).
    void limit_handles_for_testing(uint32_t end) { handle_end_ = end; }

    // SchedulerConfig::proactive_filling_reserve / _max (scheduler/state.rs:14-21).  tako's defaults are 16 / 40; this
    // class starts with proactive filling OFF (max = 0) and the embedding server switches it on.
    void set_scheduler_config(uint32_t proactive_filling_reserve, uint32_t proactive_filling_max);
    // reactor.rs:263-345 (RunningPrefilled): the worker started one of its prefilled tasks with the given variant
    void on_task_running_prefilled(TaskId task, ResourceVariantId variant);
    // on_retract_response (reactor.rs:452-498): tasks the worker gave back; returns the ComputeTasks lists for the
    // redirect targets (target worker -> [(task, variant)])
    std::map<WorkerId, std::vector<std::pair<TaskId, ResourceVariantId>>> on_retract_response(WorkerId worker, const std::vector<TaskId>& tasks);
    size_t n_prefilled(WorkerId id) const;
    const std::map<uint64_t, std::pair<WorkerId, ResourceVariantId>>& redirects() const { return redirects_; }   // SchedulerState::redirects

    size_t n_workers() const { return workers_.size(); }
    const std::vector<ResourceAmount>& free_resources(WorkerId id) const;   // SingleNodeTaskAssignment::free_resources
    const std::string& last_error() const { return last_error_; }
    hqs_stats stats() const;

private:
    struct WorkerState {
        std::vector<ResourceAmount> total, free;
        float min_utilization = 0.0f;
        std::optional<uint64_t> termination_ms;
        std::vector<std::pair<ResourceRqId, ResourceVariantId>> blocked;
    };
    struct TaskState {
        TaskId id;
        ResourceRqId rq = 0;
        Priority priority = 0;
        int64_t worker = -1;              // TaskRuntimeState::Assigned{worker_id, rv_id} (task.rs:22-43)
        ResourceVariantId variant = 0;
        bool live = false;                // in the ready set, assigned or running
        bool waiting = false;             // submitted with a dependency that has not finished yet
        int64_t prefilled_on = -1;        // TaskRuntimeState::Prefilled{worker_id}
        int64_t retracting_from = -1;     // TaskRuntimeState::Retracting{worker_id}
        bool forgotten = false;           // finished, or cancelled / failed: tako no longer knows it (retire_handles)
    };
    struct TickInput {                    // the worker view of one tick in the C ABI's form + the free vectors it returns
        std::vector<hqs_worker> hw;
        std::vector<uint64_t> free_rw, total_rw, free_after;
        std::vector<uint8_t> blocked;     // empty: no blocked request
        std::vector<WorkerId> ids;
    };
    bool tick_input(uint64_t now_ms, TickInput& in);
    void apply_free_after(const TickInput& in);
    void flush_classes();
    void flush_ready();
    void flush_graph();
    uint32_t handle_of(TaskId task);
    std::vector<uint32_t> cancel_on_device(const std::vector<uint32_t>& handles);
    int64_t leave_worker(TaskState& t);

    hqs_ctx* ctx_ = nullptr;
    uint32_t R_;
    std::map<std::string, ResourceRqId> rq_ids_;             // interning key = canonical byte string of the variants
    std::vector<hqs_class> classes_;
    bool classes_dirty_ = false;
    std::map<WorkerId, WorkerState> workers_;                // ordered by id (solver.rs:44)
    std::unordered_map<uint64_t, uint32_t> handle_of_;       // TaskId -> dense handle
    std::vector<TaskState> tasks_;                           // by handle
    std::vector<uint32_t> push_h_, push_c_;
    std::vector<uint32_t> forget_h_;                         // finished tasks: leave the device table at the next flush
    std::vector<uint64_t> push_p_;
    // graph submits batched until the next flush: handle, class, priority, dependency handles
    std::vector<uint32_t> graph_h_, graph_c_;
    std::vector<uint64_t> graph_p_;
    std::vector<std::vector<uint32_t>> graph_deps_;
    // set by the first submit with dependencies: the flush pushes the graph batch and sends finishes through
    // hqs_graph_finished (both in tako_shim_graph.cpp)
    void (GpuCore::*graph_flush_)() = nullptr;
    std::vector<hqs_assignment> out_;
    uint32_t handle_end_ = 0xFFFFFFFFu;                      // handle_of gives out handles below this
    uint32_t pf_max_ = 0;
    std::map<uint64_t, std::pair<WorkerId, ResourceVariantId>> redirects_;
    std::string last_error_;
};

}  // namespace tako_b200

extern "C" {
// Self-test of the shim on CUDA device `device` (small scenarios restated from tests/test_scheduler_sn.rs plus a
// zero-duration drain with a host-side replay of every placement).  Returns the number of failed checks.
int hqshim_selftest(int device, int verbose);
// Self-test of GpuCore::run_scheduling_grouped on CUDA device `device`: two identically loaded cores, one ticking flat and
// one grouped, through a multi-class drain with priorities and through proactive filling with retract / redirect; every
// tick's mappings must be equal, list order included, and so must the free vectors.  Returns the number of failed checks.
int hqshim_selftest_grouped(int device, int verbose);
// Self-test of GpuCore's task graphs on CUDA device `device` (tako_shim_graph.cpp): seeded random jobs with dependencies on
// earlier jobs, submitted between ticks of a zero-duration drain, with cancellations; every task runs once, never before a
// dependency that was live at its submit finished, and the host mirror's waiting set matches the device's.  Returns the
// number of failed checks.
int hqshim_selftest_graph(int device, int verbose);
// Self-test of GpuCore::on_cancel_tasks / on_task_failed on CUDA device `device` (tako_shim_graph_cancel.cpp): seeded random
// jobs with dependencies in a zero-duration drain with proactive filling on, random cancels of tasks in every state and
// failures of assigned tasks.  Every task runs once or is reported as left exactly once, the reported consumers equal the
// test's own closure, and the free vectors return to the totals.  Returns the number of failed checks.
int hqshim_selftest_graph_cancel(int device, int verbose);
// Self-test of GpuCore::retire_handles on CUDA device `device` (tako_shim_retire.cpp): two cores get the same seeded
// zero-duration drain of jobs with dependencies, proactive filling, cancels, failures and retract responses; one retires its
// forgotten handles every few ticks, the other never does.  Every WorkerTaskMapping, every cancel and failure list and the
// free vectors must be equal, and after each retire the retiring core's n_handles() must not exceed the tasks tako still
// knows.
// Returns the number of failed checks.
int hqshim_selftest_retire(int device, int verbose);
// Measuring aid (tools/grouped_probe.py): host wall time of one tick INCLUDING the construction of the per-worker lists of a
// WorkerTaskMapping, on a context the caller has loaded (handles stand in for TaskIds).  grouped = 0: hqs_tick and one map
// lookup + push_back per record of the flat stream; grouped = 1: hqs_tick_grouped and one lookup + reserved append per worker,
// as GpuCore::run_scheduling_grouped does.  Before each of the `reps` ticks the ready set is re-armed (not timed).
// out_ms[reps] receives the times, *digest a hash of the lists of the last tick (equal for both forms).  Returns an HQS_E_* code.
int hqshim_time_mapping(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                        const uint64_t* total_rw, uint32_t out_cap, int grouped, uint32_t reps, double* out_ms, uint64_t* digest);
}
