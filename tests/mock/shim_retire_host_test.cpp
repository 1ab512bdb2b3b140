// Host-logic checks of tako_b200::GpuCore::retire_handles against the test double of the C ABI (fake_hqsched_retire.cpp):
// retired TaskIds are unknown afterwards, kept ones keep their TaskIds in handle order, a started prefilled task and a
// retracting one keep their handles, later finishes, cancels and retract responses behave as on a twin core that never
// retires, handle_of throws at the end of the handle space, and the GPU self-test's drain runs against the double as well.
// Returns the number of failed checks.
#include "../../include/tako_shim.hpp"

#include <cstdio>
#include <stdexcept>

extern "C" int hqshim_selftest_retire(int device, int verbose);

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
static bool same(const WorkerTaskMapping& a, const WorkerTaskMapping& b) {
    if (a.workers.size() != b.workers.size()) return false;
    for (const auto& kv : a.workers) {
        auto it = b.workers.find(kv.first);
        if (it == b.workers.end() || kv.second.assigned != it->second.assigned || kv.second.prefills != it->second.prefills ||
            kv.second.retracts != it->second.retracts)
            return false;
    }
    return true;
}

int main() {
    const Priority p = priority_from_user(0);
    {   // graph core: finished and cancelled tasks go, waiting, ready, running and announced ones stay
        GpuCore a(1, 0), b(1, 0);
        for (GpuCore* c : {&a, &b}) {
            const ResourceRqId c1 = c->get_or_create_resource_rq_id(cpus(1));
            c->on_new_worker(1, {2 * FRACTIONS_PER_UNIT});
            c->on_new_tasks(std::vector<NewTask>{{TaskId{1, 1}, c1, p, {}}, {TaskId{1, 2}, c1, p, {}},
                                                   {TaskId{1, 3}, c1, p, {TaskId{1, 1}}}, {TaskId{1, 4}, c1, p, {TaskId{1, 3}}},
                                                   {TaskId{1, 5}, c1, p, {}}, {TaskId{1, 6}, c1, p, {TaskId{1, 5}}}});
        }
        check(same(a.run_scheduling(), b.run_scheduling()), "first tick");
        for (GpuCore* c : {&a, &b}) {
            c->on_task_finished(TaskId{1, 1});                     // 1.3 becomes ready
            c->on_cancel_tasks({TaskId{1, 5}});                    // 1.5 and its consumer 1.6 leave
            c->on_new_tasks(std::vector<TaskId>{TaskId{2, 1}});    // announced, never made ready yet
        }
        check(a.n_handles() == 7, "seven handles before the retire");
        check(a.retire_handles() == 3 && a.n_handles() == 4, "1.1, 1.5 and 1.6 retired: 1.2, 1.3, 1.4 and 2.1 stay");
        check(a.n_waiting() == b.n_waiting() && a.n_waiting() == 1, "1.4 still waits");
        check(a.retire_handles() == 0 && a.n_handles() == 4, "a second retire retires nothing");
        for (GpuCore* c : {&a, &b}) c->add_ready_task(TaskId{2, 1}, 0, p);
        const WorkerTaskMapping ma = a.run_scheduling(), mb = b.run_scheduling();
        check(same(ma, mb) && ma.n_assigned() == 1, "the kept tasks keep their TaskIds: 1.3 runs");
        for (GpuCore* c : {&a, &b}) {
            c->on_task_finished(TaskId{1, 1});                     // retired on a: unknown; finished already on b
            c->on_task_finished(TaskId{1, 2});
            c->on_task_finished(TaskId{1, 3});                     // releases 1.4
        }
        check(a.free_resources(1) == b.free_resources(1), "finishes of kept and retired tasks agree");
        check(same(a.run_scheduling(), b.run_scheduling()), "the released consumer runs on both");
        const CancelledTasks ca = a.on_cancel_tasks({TaskId{1, 6}, TaskId{1, 4}, TaskId{2, 1}});
        const CancelledTasks cb = b.on_cancel_tasks({TaskId{1, 6}, TaskId{1, 4}, TaskId{2, 1}});
        check(ca.cancelled == cb.cancelled && ca.messages == cb.messages && ca.cancelled.size() == 2, "cancels agree");
        check(a.retire_handles() == 4 && a.n_handles() == 0, "everything is forgotten: the table is empty");
        for (GpuCore* c : {&a, &b}) c->on_new_tasks(std::vector<NewTask>{{TaskId{3, 1}, 0, p, {TaskId{1, 4}}}});
        check(same(a.run_scheduling(), b.run_scheduling()) && a.n_handles() == 1, "a new task after an empty table");
    }
    {   // proactive filling: a started prefilled task and a retracting one keep their handles
        GpuCore a(1, 0), b(1, 0);
        for (GpuCore* c : {&a, &b}) {
            const ResourceRqId c1 = c->get_or_create_resource_rq_id(cpus(1));
            c->set_scheduler_config(0, 1);
            c->on_new_worker(1, {1 * FRACTIONS_PER_UNIT});
            c->on_new_worker(2, {1 * FRACTIONS_PER_UNIT});
            for (uint32_t t = 1; t <= 6; ++t) c->add_ready_task(TaskId{1, t}, c1, p);
        }
        WorkerTaskMapping m = a.run_scheduling();
        check(same(m, b.run_scheduling()) && m.n_assigned() == 2, "two assigned, prefills behind them");
        std::vector<TaskId> pf;
        for (const auto& kv : m.workers)
            for (const TaskId& t : kv.second.prefills) pf.push_back(t);
        check(pf.size() == 2, "two prefilled");
        for (GpuCore* c : {&a, &b}) {
            for (const auto& kv : m.workers)
                for (const auto& tv : kv.second.assigned) c->on_task_finished(tv.first);
            c->on_task_running_prefilled(pf[0], 0);                // removed from the ready set, still running
        }
        check(a.retire_handles() == 2, "the two finished tasks are retired");
        check(same(a.run_scheduling(), b.run_scheduling()), "the tick after the retire");
        for (GpuCore* c : {&a, &b}) c->on_task_finished(pf[0]);
        check(a.free_resources(1) == b.free_resources(1) && a.free_resources(2) == b.free_resources(2),
              "the started prefilled task finishes with its resources on both");
        a.retire_handles();
        check(same(a.run_scheduling(), b.run_scheduling()), "and the tick after that");
        check(a.redirects() == b.redirects(), "the redirects agree");
    }
    {   // the end of the handle space
        GpuCore c(1, 0);
        c.limit_handles_for_testing(2);
        c.on_new_tasks(std::vector<TaskId>{TaskId{1, 1}, TaskId{1, 2}});
        bool threw = false;
        try { c.on_new_tasks(std::vector<TaskId>{TaskId{1, 3}}); } catch (const std::length_error&) { threw = true; }
        check(threw && c.n_handles() == 2, "handle_of throws instead of wrapping");
    }
    check(hqshim_selftest_retire(0, 0) == 0, "the retire self-test's drain against the double");
    std::fprintf(stderr, "shim retire host test: %d failed\n", failed);
    return failed;
}
