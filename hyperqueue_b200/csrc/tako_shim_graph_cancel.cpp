// tako_shim_graph_cancel.cpp — GpuCore::on_cancel_tasks / on_task_failed (include/tako_shim.hpp) and their GPU self-test.  A
// core that has submitted tasks with dependencies removes the named tasks with their waiting consumers in one
// hqs_graph_cancel; any other core removes the named tasks with hqs_ready_remove, as remove_ready_task does.
#include "../../include/tako_shim.hpp"

#include <algorithm>
#include <cstdio>
#include <exception>
#include <map>
#include <set>
#include <stdexcept>
#include <vector>

namespace tako_b200 {

// The handles that left the device table: on a graph core the named VALID ones and all their waiting consumers, ascending.
std::vector<uint32_t> GpuCore::cancel_on_device(const std::vector<uint32_t>& handles) {
    if (handles.empty()) return {};
    if (!graph_flush_) {
        if (hqs_ready_remove(ctx_, (uint32_t)handles.size(), handles.data()) != HQS_OK) {
            last_error_ = hqs_last_error(ctx_);
            std::fprintf(stderr, "[tako_b200] hqs_ready_remove: %s\n", last_error_.c_str());
        }
        return {};
    }
    const uint32_t* left = nullptr;
    uint32_t n = 0;
    if (hqs_graph_cancel(ctx_, (uint32_t)handles.size(), handles.data(), &left, &n) != HQS_OK) {
        last_error_ = hqs_last_error(ctx_);
        throw std::runtime_error("hqs_graph_cancel: " + last_error_);
    }
    return std::vector<uint32_t>(left, left + n);
}

// The worker side of a task that leaves (reactor.rs:612-659, 720-760): an assigned or running task's resources go back
// (Worker::remove_sn_task), a prefilled task is no longer held, a retracting task's redirect is dropped and the redirect
// target's resources come back (try_remove_redirection, reactor.rs:582-594).  Returns the worker a CancelTasks message
// goes to, -1 for none.
int64_t GpuCore::leave_worker(TaskState& t) {
    int64_t to = -1;
    if (t.retracting_from >= 0) {
        to = t.retracting_from;
        redirects_.erase(t.id.as_u64());
    } else if (t.worker >= 0) {
        to = t.worker;
    } else if (t.prefilled_on >= 0) {
        to = t.prefilled_on;
    }
    if (t.worker >= 0) {
        auto wit = workers_.find((WorkerId)t.worker);
        if (wit != workers_.end()) {
            WorkerState& w = wit->second;
            const hqs_variant& hv = classes_[t.rq].variants[t.variant];
            for (uint32_t r = 0; r < R_; ++r) {
                if ((hv.all_mask >> r) & 1) w.free[r] = w.total[r];
                else if (hv.amount[r] && w.free[r] != HQS_AMOUNT_MAX) w.free[r] += hv.amount[r];
            }
        }
    }
    t.worker = -1;
    t.prefilled_on = -1;
    t.retracting_from = -1;
    t.live = false;
    t.waiting = false;
    t.forgotten = true;
    return to;
}

CancelledTasks GpuCore::on_cancel_tasks(const std::vector<TaskId>& tasks) {
    flush_ready();                       // the device holds every submit and every finish
    CancelledTasks out;
    std::vector<uint32_t> named;
    std::set<uint32_t> left;
    for (const TaskId& id : tasks) {
        auto it = handle_of_.find(id.as_u64());
        if (it == handle_of_.end()) continue;                   // "Task is not here"
        TaskState& t = tasks_[it->second];
        if (!t.live && !t.waiting) continue;                    // finished or cancelled already
        const int64_t to = leave_worker(t);
        if (to >= 0) out.messages[(WorkerId)to].push_back(id);
        named.push_back(it->second);
        left.insert(it->second);
    }
    for (uint32_t h : cancel_on_device(named)) {
        tasks_[h].live = tasks_[h].waiting = false;             // consumers: waiting, so held by no worker
        tasks_[h].forgotten = true;
        left.insert(h);
    }
    for (uint32_t h : left) out.cancelled.push_back(tasks_[h].id);
    std::sort(out.cancelled.begin(), out.cancelled.end());
    return out;
}

std::vector<TaskId> GpuCore::on_task_failed(TaskId task) {
    flush_ready();
    auto it = handle_of_.find(task.as_u64());
    if (it == handle_of_.end()) return {};                      // "Unknown task failed"
    const uint32_t h = it->second;
    TaskState& t = tasks_[h];
    if (!t.live && !t.waiting) return {};
    leave_worker(t);                                            // no message: the worker reported the failure
    std::vector<TaskId> consumers;
    for (uint32_t c : cancel_on_device({h}))
        if (c != h) {
            tasks_[c].live = tasks_[c].waiting = false;
            tasks_[c].forgotten = true;
            consumers.push_back(tasks_[c].id);
        }
    std::sort(consumers.begin(), consumers.end());
    return consumers;
}

}  // namespace tako_b200

using namespace tako_b200;

// A zero-duration drain on the GPU with proactive filling on: seeded random jobs whose tasks depend on earlier tasks are
// submitted between ticks.  Between a tick and the finishes some assigned tasks fail and some tasks are cancelled: waiting,
// ready, prefilled, assigned and retracting ones, plus finished and unknown TaskIds.  The test keeps its own consumer map and
// checks each call's list against its own closure.
extern "C" int hqshim_selftest_graph_cancel(int device, int verbose) {
    int failed = 0;
    auto check = [&](bool ok, const char* what) {
        if (!ok) { ++failed; std::fprintf(stderr, "[shim graph cancel selftest] FAILED: %s\n", what); }
        else if (verbose) std::fprintf(stderr, "[shim graph cancel selftest] ok: %s\n", what);
    };
    try {
        GpuCore core(1, device);
        core.set_scheduler_config(1, 2);
        std::vector<ResourceRqId> rqs;
        for (uint64_t c = 1; c <= 3; ++c) {
            ResourceRequest rq;
            rq.entries.push_back({0, false, c * FRACTIONS_PER_UNIT});
            rqs.push_back(core.get_or_create_resource_rq_id(ResourceRequestVariants{{rq}}));
        }
        core.on_new_worker(50, {12 * FRACTIONS_PER_UNIT});
        core.on_new_worker(51, {8 * FRACTIONS_PER_UNIT});
        uint64_t x = 0x2545F4914F6CDD1Dull;
        auto rnd = [&](uint64_t n) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x % n; };
        auto tid = [](uint64_t v) { return TaskId{(uint32_t)(v >> 32), (uint32_t)v}; };
        enum { ALIVE, DONE, LEFT };
        std::map<uint64_t, int> state;
        std::map<uint64_t, int> runs, leaves;
        std::map<uint64_t, std::vector<uint64_t>> consumers;     // only edges made while the producer was alive
        std::vector<uint64_t> all;
        std::map<uint64_t, WorkerId> prefilled;                   // prefilled at some tick (a superset: retracts are not erased)
        bool lists_ok = true, fail_ok = true, msgs_ok = true;
        size_t n_cancel_named = 0, n_failed = 0, n_consumers = 0;
        auto closure = [&](const std::vector<uint64_t>& named) {
            std::set<uint64_t> out;
            std::vector<uint64_t> stack;
            for (uint64_t v : named)
                if (state.count(v) && state[v] == ALIVE && out.insert(v).second) stack.push_back(v);
            while (!stack.empty()) {
                const uint64_t v = stack.back();
                stack.pop_back();
                for (uint64_t c : consumers[v])
                    if (state[c] == ALIVE && out.insert(c).second) stack.push_back(c);
            }
            return out;
        };
        auto mark_left = [&](const std::vector<TaskId>& ids) {
            for (const TaskId& t : ids) { state[t.as_u64()] = LEFT; ++leaves[t.as_u64()]; }
        };
        auto cancel = [&](const std::vector<uint64_t>& named, const std::set<uint64_t>& held) {
            const std::set<uint64_t> want = closure(named);
            std::vector<TaskId> ids;
            for (uint64_t v : named) ids.push_back(tid(v));
            const CancelledTasks r = core.on_cancel_tasks(ids);
            std::set<uint64_t> got;
            for (const TaskId& t : r.cancelled) got.insert(t.as_u64());
            lists_ok &= got == want && got.size() == r.cancelled.size();
            for (const auto& kv : r.messages)     // only named tasks that a worker holds
                for (const TaskId& t : kv.second)
                    msgs_ok &= held.count(t.as_u64()) != 0 && std::find(named.begin(), named.end(), t.as_u64()) != named.end();
            mark_left(r.cancelled);
            n_cancel_named += named.size();
        };
        uint32_t job = 1;
        size_t submitted = 0;
        for (int tick = 0; tick < 300; ++tick) {
            if (tick < 100 && rnd(3) != 0) {
                const uint32_t k = 1 + (uint32_t)rnd(25);
                std::vector<NewTask> batch;
                for (uint32_t t = 1; t <= k; ++t) {
                    NewTask nt{TaskId{job, t}, rqs[rnd(rqs.size())], priority_from_user((int32_t)rnd(3)), {}};
                    for (uint32_t j = 0, nd = (uint32_t)rnd(4); j < nd; ++j) {
                        TaskId d;
                        if (rnd(2) == 0 && t > 1) d = TaskId{job, 1 + (uint32_t)rnd(t - 1)};
                        else if (!all.empty()) d = tid(all[all.size() - 1 - rnd(std::min<size_t>(all.size(), 150))]);
                        else continue;
                        if (std::find(nt.deps.begin(), nt.deps.end(), d) == nt.deps.end()) nt.deps.push_back(d);
                    }
                    const uint64_t me = nt.id.as_u64();
                    for (const TaskId& d : nt.deps) {
                        auto s = state.find(d.as_u64());
                        if (s != state.end() && s->second == ALIVE) consumers[d.as_u64()].push_back(me);
                    }
                    state[me] = ALIVE;
                    batch.push_back(nt);
                }
                for (const NewTask& nt : batch) all.push_back(nt.id.as_u64());
                submitted += k;
                core.on_new_tasks(batch);
                ++job;
            }
            const WorkerTaskMapping m = core.run_scheduling();
            std::set<uint64_t> held;                            // tasks some worker holds: assigned, prefilled, retracting
            std::vector<uint64_t> running;
            std::vector<std::pair<WorkerId, uint64_t>> retracting;
            for (const auto& kv : m.workers) {
                for (const auto& tv : kv.second.assigned) { running.push_back(tv.first.as_u64()); held.insert(tv.first.as_u64()); }
                for (const TaskId& t : kv.second.retracts) { retracting.push_back({kv.first, t.as_u64()}); held.insert(t.as_u64()); }
            }
            for (const auto& kv : m.workers)
                for (const TaskId& t : kv.second.prefills) prefilled[t.as_u64()] = kv.first;
            for (const auto& kv : prefilled) held.insert(kv.first);
            if (!all.empty() && rnd(3) == 0) {                  // a cancel of tasks in any state
                std::vector<uint64_t> named;
                for (int j = 0, k = 1 + (int)rnd(3); j < k; ++j) named.push_back(all[rnd(all.size())]);
                if (!running.empty()) named.push_back(running[rnd(running.size())]);
                if (!retracting.empty()) named.push_back(retracting[rnd(retracting.size())].second);
                if (rnd(4) == 0) named.push_back(TaskId{9999, 1}.as_u64());
                cancel(named, held);
            }
            if (!running.empty() && rnd(3) == 0) {             // a failure of an assigned task
                const uint64_t v = running[rnd(running.size())];
                if (state[v] == ALIVE) {
                    std::set<uint64_t> want = closure({v});
                    want.erase(v);
                    const std::vector<TaskId> cons = core.on_task_failed(tid(v));
                    std::set<uint64_t> got;
                    for (const TaskId& t : cons) got.insert(t.as_u64());
                    fail_ok &= got == want && got.size() == cons.size();
                    mark_left(cons);
                    mark_left({tid(v)});
                    ++n_failed;
                    n_consumers += cons.size();
                }
            }
            for (const auto& wr : retracting) {                 // the retracted tasks come back and run on their targets
                if (state[wr.second] != ALIVE) continue;
                for (const auto& kv : core.on_retract_response(wr.first, {tid(wr.second)}))
                    for (const auto& tv : kv.second) running.push_back(tv.first.as_u64());
            }
            for (uint64_t v : running) {
                if (state[v] != ALIVE) continue;
                state[v] = DONE;
                ++runs[v];
                core.on_task_finished(tid(v));
            }
            bool alive = false;
            for (const auto& kv : state) alive |= kv.second == ALIVE;
            if (tick >= 100 && !alive) break;
        }
        // whatever is still prefilled or waiting at the end is cancelled, so every task is accounted for
        {
            std::vector<uint64_t> rest;
            for (const auto& kv : state)
                if (kv.second == ALIVE) rest.push_back(kv.first);
            cancel(rest, std::set<uint64_t>(rest.begin(), rest.end()));
        }
        bool once = true;
        for (uint64_t v : all) once &= runs[v] + leaves[v] == 1;
        check(once, "every task runs once or is reported as left exactly once");
        check(lists_ok, "on_cancel_tasks lists the named live tasks and their transitive waiting consumers");
        check(fail_ok, "on_task_failed lists the failed task's transitive waiting consumers");
        check(msgs_ok, "CancelTasks messages name only tasks a worker holds");
        check(core.n_waiting() == 0, "nothing waits at the end");
        check(core.redirects().empty(), "no redirect is left");
        check(core.free_resources(50)[0] == 12 * FRACTIONS_PER_UNIT && core.free_resources(51)[0] == 8 * FRACTIONS_PER_UNIT,
              "the workers' resources are all back");
        check(n_cancel_named > 0 && n_failed > 0 && n_consumers > 0, "cancels, failures and reported consumers happened");
        if (verbose)
            std::fprintf(stderr, "[shim graph cancel selftest] %zu tasks, %zu named in cancels, %zu failures with %zu consumers\n",
                         submitted, n_cancel_named, n_failed, n_consumers);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "[shim graph cancel selftest] exception: %s\n", e.what());
        ++failed;
    }
    return failed;
}
