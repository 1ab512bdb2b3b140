// Host-logic checks of tako_b200::GpuCore's task graphs against the test double of the C ABI (fake_hqsched_graph.cpp): dependency
// resolution at submit (unknown, finished and cancelled producers are dropped), the batched graph push at the flush, finishes
// through hqs_graph_finished once a core has submitted a task with dependencies, released tasks becoming schedulable, and
// cancellation before and after the flush.  Returns the number of failed checks.
#include "../../include/tako_shim.hpp"

#include <cstdio>
#include <set>

using namespace tako_b200;

static int failed = 0;
static void check(bool ok, const char* what) {
    if (!ok) { ++failed; std::fprintf(stderr, "FAILED: %s\n", what); }
}
static ResourceRequestVariants cpus(uint64_t n) {
    ResourceRequest rq;
    rq.entries.push_back({0, false, n * FRACTIONS_PER_UNIT});
    return ResourceRequestVariants{{rq}};
}
static std::set<uint64_t> assigned(const WorkerTaskMapping& m) {
    std::set<uint64_t> out;
    for (const auto& kv : m.workers)
        for (const auto& tv : kv.second.assigned) out.insert(tv.first.as_u64());
    return out;
}
static uint64_t id(uint32_t job, uint32_t task) { return TaskId{job, task}.as_u64(); }

int main() {
    {   // a chain and a join over two submits; finishes release consumers only when their last producer is done
        GpuCore core(1, 0);
        const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
        core.on_new_worker(1, {8 * FRACTIONS_PER_UNIT});
        const Priority p = priority_from_user(0);
        core.on_new_tasks(std::vector<NewTask>{{TaskId{1, 1}, c1, p, {}}, {TaskId{1, 2}, c1, p, {}}});
        core.on_new_tasks(std::vector<NewTask>{{TaskId{2, 2}, c1, p, {TaskId{2, 1}}},                 // same submit, earlier TaskId
                                               {TaskId{2, 1}, c1, p, {TaskId{1, 1}, TaskId{1, 2}}},
                                               {TaskId{2, 3}, c1, p, {TaskId{9, 9}}},                  // unknown: dropped
                                               {TaskId{2, 4}, c1, p, {TaskId{2, 5}}}});               // later TaskId: dropped
        check(core.n_waiting() == 2, "two tasks wait for dependencies");
        check(core.stats().n_groups == 0, "graph submits are batched until the flush");
        WorkerTaskMapping m = core.run_scheduling();
        check(core.stats().n_groups == 6, "one graph push of six tasks");
        check(assigned(m) == std::set<uint64_t>{id(1, 1), id(1, 2), id(2, 3), id(2, 4)}, "the four ready tasks run");
        core.on_task_finished(TaskId{1, 1});
        m = core.run_scheduling();
        check(m.n_assigned() == 0 && core.n_waiting() == 2, "one of two producers finished: the join still waits");
        check(core.stats().n_levels == 1 && core.stats().n_segments == 0, "finishes go through hqs_graph_finished");
        core.on_task_finished(TaskId{1, 2});
        m = core.run_scheduling();
        check(assigned(m) == std::set<uint64_t>{id(2, 1)} && core.n_waiting() == 1, "the join is released");
        core.on_task_finished(TaskId{2, 1});
        m = core.run_scheduling();
        check(assigned(m) == std::set<uint64_t>{id(2, 2)} && core.n_waiting() == 0, "the chain's last task is released");
        core.on_task_finished(TaskId{2, 2});
        check(core.free_resources(1)[0] == 6 * FRACTIONS_PER_UNIT, "released tasks return their resources when they finish");
        // a dependency on a finished task is dropped: ready at once
        core.on_new_tasks(std::vector<NewTask>{{TaskId{3, 1}, c1, p, {TaskId{2, 2}}}});
        check(core.n_waiting() == 0, "a finished producer does not count");
        check(assigned(core.run_scheduling()) == std::set<uint64_t>{id(3, 1)}, "and the task runs");
    }
    {   // cancellation: before the flush the task never reaches the device and its consumers do not wait for it; after the
        // flush it leaves the device table and its consumers are cancelled by the host too
        GpuCore core(1, 0);
        const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
        core.on_new_worker(1, {1 * FRACTIONS_PER_UNIT});
        const Priority p = priority_from_user(0);
        core.on_new_tasks(std::vector<NewTask>{{TaskId{1, 1}, c1, p, {}}, {TaskId{1, 2}, c1, p, {TaskId{1, 1}}}});
        core.remove_ready_task(TaskId{1, 1});
        WorkerTaskMapping m = core.run_scheduling();
        check(core.stats().n_groups == 1 && core.stats().n_segments == 0, "the cancelled task is not pushed");
        check(assigned(m) == std::set<uint64_t>{id(1, 2)} && core.n_waiting() == 0, "its consumer is ready at once");
        core.on_new_tasks(std::vector<NewTask>{{TaskId{2, 1}, c1, p, {TaskId{1, 2}}}, {TaskId{2, 2}, c1, p, {TaskId{2, 1}}}});
        m = core.run_scheduling();
        check(m.n_assigned() == 0 && core.n_waiting() == 2, "both wait on the running task");
        core.remove_ready_task(TaskId{2, 1});
        core.remove_ready_task(TaskId{2, 2});
        check(core.stats().n_segments == 2 && core.n_waiting() == 0, "a flushed waiting task is cancelled on the device");
        core.on_task_finished(TaskId{1, 2});
        m = core.run_scheduling();
        check(m.n_assigned() == 0, "cancelled consumers are not released");
        check(core.free_resources(1)[0] == 1 * FRACTIONS_PER_UNIT, "the finished task returned its cpu");
    }
    {   // a core without dependencies keeps removing finished tasks with hqs_ready_remove
        GpuCore core(1, 0);
        const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
        core.on_new_worker(1, {1 * FRACTIONS_PER_UNIT});
        core.add_ready_task(TaskId{1, 1}, c1, 0);
        core.run_scheduling();
        core.on_task_finished(TaskId{1, 1});
        core.run_scheduling();
        check(core.stats().n_segments == 1 && core.stats().n_levels == 0, "plain cores do not use the graph calls");
    }
    std::fprintf(stderr, "shim graph host test: %d failed\n", failed);
    return failed;
}
