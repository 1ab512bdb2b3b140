// Host-logic checks of tako_b200::GpuCore::on_cancel_tasks / on_task_failed against the test double of the C ABI
// (fake_hqsched_graph_cancel.cpp): cancels before and after the flush, the CancelTasks lists per worker for assigned,
// prefilled and retracting tasks, resources coming back, failures reporting their consumers, and nothing left waiting after
// the roots of every job are cancelled.  Returns the number of failed checks.
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
static std::vector<uint64_t> ids(const std::vector<TaskId>& v) {
    std::vector<uint64_t> out;
    for (const TaskId& t : v) out.push_back(t.as_u64());
    return out;
}
static uint64_t id(uint32_t job, uint32_t task) { return TaskId{job, task}.as_u64(); }

int main() {
    const Priority p = priority_from_user(0);
    {   // before the flush: the cancel flushes the submit first, so the chain's consumers leave with their root
        GpuCore core(1, 0);
        const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
        core.on_new_worker(1, {4 * FRACTIONS_PER_UNIT});
        core.on_new_tasks(std::vector<NewTask>{{TaskId{1, 1}, c1, p, {}}, {TaskId{1, 2}, c1, p, {TaskId{1, 1}}},
                                               {TaskId{1, 3}, c1, p, {TaskId{1, 2}}}, {TaskId{1, 4}, c1, p, {}}});
        check(core.n_waiting() == 2, "two tasks wait");
        const CancelledTasks r = core.on_cancel_tasks({TaskId{1, 1}, TaskId{7, 7}, TaskId{1, 1}});
        check(ids(r.cancelled) == std::vector<uint64_t>{id(1, 1), id(1, 2), id(1, 3)}, "before the flush: the root and its chain");
        check(r.messages.empty() && core.n_waiting() == 0, "nothing was held by a worker, nothing waits");
        const WorkerTaskMapping m = core.run_scheduling();
        check(m.n_assigned() == 1 && m.workers.at(1).assigned[0].first.as_u64() == id(1, 4), "only the unrelated task runs");
        // after the flush: a consumer of a running task is cancelled with it, and the running task's cpu comes back
        core.on_new_tasks(std::vector<NewTask>{{TaskId{2, 1}, c1, p, {TaskId{1, 4}}}, {TaskId{2, 2}, c1, p, {TaskId{2, 1}}}});
        core.run_scheduling();
        check(core.free_resources(1)[0] == 3 * FRACTIONS_PER_UNIT && core.n_waiting() == 2, "after the flush: two wait");
        const CancelledTasks q = core.on_cancel_tasks({TaskId{1, 4}});
        check(ids(q.cancelled) == std::vector<uint64_t>{id(1, 4), id(2, 1), id(2, 2)}, "the running task and its consumers");
        check(q.messages.size() == 1 && ids(q.messages.at(1)) == std::vector<uint64_t>{id(1, 4)}, "CancelTasks to its worker");
        check(core.free_resources(1)[0] == 4 * FRACTIONS_PER_UNIT && core.n_waiting() == 0, "its cpu is back");
        check(core.on_cancel_tasks({TaskId{1, 4}}).cancelled.empty(), "a second cancel finds nothing");
    }
    {   // assigned, prefilled and retracting tasks: messages per worker in the order named, resources back
        GpuCore core(1, 0);
        const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
        core.on_new_worker(1, {1 * FRACTIONS_PER_UNIT});
        core.on_new_worker(2, {1 * FRACTIONS_PER_UNIT});
        core.set_scheduler_config(0, 1);
        std::vector<NewTask> job;
        for (uint32_t t = 1; t <= 4; ++t) job.push_back({TaskId{1, t}, c1, p, {}});
        core.on_new_tasks(job);
        WorkerTaskMapping m = core.run_scheduling();
        std::map<uint64_t, WorkerId> where, pf;
        for (const auto& kv : m.workers) {
            for (const auto& tv : kv.second.assigned) where[tv.first.as_u64()] = kv.first;
            for (const TaskId& t : kv.second.prefills) pf[t.as_u64()] = kv.first;
        }
        check(where.size() == 2 && pf.size() == 2, "two tasks assigned, two prefilled");
        const uint64_t a0 = where.begin()->first, a1 = std::next(where.begin())->first;
        std::vector<NewTask> cons{{TaskId{2, 1}, c1, p, {TaskId{1, (uint32_t)a1}}}};   // one consumer of each task but a0
        for (const auto& kv : pf) cons.push_back({TaskId{2, (uint32_t)cons.size() + 1}, c1, p, {TaskId{1, (uint32_t)kv.first}}});
        cons.push_back({TaskId{2, 9}, c1, p, {TaskId{2, 1}}});
        core.on_new_tasks(cons);
        core.on_task_finished(TaskId{1, (uint32_t)a0});         // frees a worker: the next tick takes a prefilled task
        m = core.run_scheduling();
        uint64_t retracting = 0;
        WorkerId from = 0;
        for (const auto& kv : m.workers)
            for (const TaskId& t : kv.second.retracts) { retracting = t.as_u64(); from = kv.first; }
        check(retracting != 0 && core.redirects().size() == 1, "a prefilled task is retracting");
        uint64_t still_pf = 0;
        for (const auto& kv : pf)
            if (kv.first != retracting) still_pf = kv.first;
        const std::vector<TaskId> named{TaskId{1, (uint32_t)still_pf}, TaskId{1, (uint32_t)a1}, TaskId{1, (uint32_t)retracting}};
        const CancelledTasks r = core.on_cancel_tasks(named);
        std::map<WorkerId, std::vector<uint64_t>> want;
        want[pf[still_pf]].push_back(still_pf);
        want[where[a1]].push_back(a1);
        want[from].push_back(retracting);
        std::map<WorkerId, std::vector<uint64_t>> got;
        for (const auto& kv : r.messages) got[kv.first] = ids(kv.second);
        check(got == want, "CancelTasks: the prefilled task's holder, the assigned task's worker, the retract source");
        check(r.cancelled.size() == 7 && core.n_waiting() == 0, "three named tasks and their four consumers left");
        check(core.redirects().empty() && core.n_prefilled(1) + core.n_prefilled(2) == 0, "no redirect, nothing prefilled");
        check(core.free_resources(1)[0] == FRACTIONS_PER_UNIT && core.free_resources(2)[0] == FRACTIONS_PER_UNIT,
              "the assigned task's and the redirect target's cpus are back");
    }
    {   // a failure: its transitive consumers, no message, its cpu back
        GpuCore core(1, 0);
        const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
        core.on_new_worker(1, {2 * FRACTIONS_PER_UNIT});
        core.on_new_tasks(std::vector<NewTask>{{TaskId{1, 1}, c1, p, {}}, {TaskId{1, 2}, c1, p, {TaskId{1, 1}}},
                                               {TaskId{1, 3}, c1, p, {TaskId{1, 1}, TaskId{1, 2}}}, {TaskId{1, 4}, c1, p, {}},
                                               {TaskId{1, 5}, c1, p, {TaskId{1, 4}}}});
        core.run_scheduling();
        check(core.free_resources(1)[0] == 0, "two tasks run");
        check(ids(core.on_task_failed(TaskId{1, 1})) == std::vector<uint64_t>{id(1, 2), id(1, 3)}, "the failure's consumers");
        check(core.free_resources(1)[0] == FRACTIONS_PER_UNIT && core.n_waiting() == 1, "its cpu is back; 1.5 still waits");
        check(core.on_task_failed(TaskId{1, 2}).empty(), "a consumer that left cannot fail");
    }
    {   // cancelling the roots of every job leaves nothing waiting
        GpuCore core(1, 0);
        const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
        core.on_new_worker(1, {1 * FRACTIONS_PER_UNIT});
        std::vector<TaskId> roots;
        for (uint32_t j = 1; j <= 5; ++j) {
            std::vector<NewTask> job{{TaskId{j, 1}, c1, p, {}}};
            for (uint32_t t = 2; t <= 6 * j; ++t) job.push_back({TaskId{j, t}, c1, p, {TaskId{j, t / 2}, TaskId{j, t - 1}}});
            core.on_new_tasks(job);
            roots.push_back(TaskId{j, 1});
            if (j == 3) core.run_scheduling();
        }
        check(core.n_waiting() > 0, "the jobs wait on their roots");
        const CancelledTasks r = core.on_cancel_tasks(roots);
        check(r.cancelled.size() == 6 * (1 + 2 + 3 + 4 + 5) && core.n_waiting() == 0, "every task left, nothing waits");
    }
    {   // a core without dependencies cancels with hqs_ready_remove and reports no consumers
        GpuCore core(1, 0);
        const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
        core.on_new_worker(1, {1 * FRACTIONS_PER_UNIT});
        core.add_ready_task(TaskId{1, 1}, c1, p);
        core.add_ready_task(TaskId{1, 2}, c1, p);
        core.run_scheduling();
        const CancelledTasks r = core.on_cancel_tasks({TaskId{1, 2}, TaskId{1, 1}});
        check(ids(r.cancelled) == std::vector<uint64_t>{id(1, 1), id(1, 2)} && r.messages.size() == 1, "both leave, one ran");
        check(core.stats().n_segments == 2 && core.free_resources(1)[0] == FRACTIONS_PER_UNIT, "hqs_ready_remove of both, cpu back");
        check(core.on_task_failed(TaskId{1, 1}).empty(), "no consumers on a plain core");
    }
    std::fprintf(stderr, "shim graph cancel host test: %d failed\n", failed);
    return failed;
}
