// tako_shim_graph.cpp — GpuCore's task graphs (on_new_tasks with dependencies, include/tako_shim.hpp) and their GPU
// self-test.  Only a graph submit makes a core's flush come here, so tako_shim.cpp itself calls no graph entry point of the
// C ABI: a host that never submits dependencies links without them.
#include "../../include/tako_shim.hpp"

#include <algorithm>
#include <cstdio>
#include <exception>
#include <map>
#include <set>
#include <stdexcept>
#include <vector>

namespace tako_b200 {

// Dependencies are resolved to handles here and filtered again at the flush (a producer cancelled in between is dropped there),
// so every dependency the flush sends is VALID on the device when the batch is pushed: the host and the device agree on which
// tasks wait.  Handles are never re-used, so a finished handle never aliases a new task.
void GpuCore::on_new_tasks(std::vector<NewTask> tasks) {
    std::sort(tasks.begin(), tasks.end(), [](const NewTask& a, const NewTask& b) { return a.id.as_u64() < b.id.as_u64(); });
    for (const NewTask& t : tasks)
        if (t.rq >= classes_.size()) throw std::invalid_argument("unknown resource request id");
    graph_flush_ = &GpuCore::flush_graph;
    for (NewTask& t : tasks) {
        const uint32_t h = handle_of(t.id);
        std::vector<uint32_t> deps;
        for (const TaskId& d : t.deps) {
            auto it = handle_of_.find(d.as_u64());
            if (it == handle_of_.end() || it->second == h) continue;
            const TaskState& p = tasks_[it->second];
            if ((p.live || p.waiting) && std::find(deps.begin(), deps.end(), it->second) == deps.end()) deps.push_back(it->second);
        }
        TaskState& s = tasks_[h];
        s.rq = t.rq; s.priority = t.priority; s.worker = -1;
        s.live = deps.empty(); s.waiting = !deps.empty();
        graph_h_.push_back(h); graph_c_.push_back(t.rq); graph_p_.push_back(t.priority);
        graph_deps_.push_back(std::move(deps));
    }
}

// The flush of a core that has submitted tasks with dependencies: ready tasks first, then the graph batch (its dependencies
// on them are VALID by then), then the finished tasks, which release their consumers.
void GpuCore::flush_graph() {
    flush_classes();
    if (!push_h_.empty()) {
        const int rc = hqs_ready_push(ctx_, (uint32_t)push_h_.size(), push_h_.data(), push_c_.data(), push_p_.data());
        if (rc != HQS_OK) { last_error_ = hqs_last_error(ctx_); throw std::runtime_error("hqs_ready_push: " + last_error_); }
        push_h_.clear(); push_c_.clear(); push_p_.clear();
    }
    if (!graph_h_.empty()) {
        std::vector<uint32_t> off(1, 0), deps;
        size_t expect_ready = 0;
        for (size_t i = 0; i < graph_h_.size(); ++i) {
            for (uint32_t d : graph_deps_[i])
                if (tasks_[d].live || tasks_[d].waiting) deps.push_back(d);   // finished or cancelled since the submit: dropped
            off.push_back((uint32_t)deps.size());
            TaskState& t = tasks_[graph_h_[i]];
            t.waiting = off[i + 1] != off[i];
            t.live = !t.waiting;
            expect_ready += t.live ? 1 : 0;
        }
        uint32_t n_ready = 0;
        const int rc = hqs_graph_push(ctx_, (uint32_t)graph_h_.size(), graph_h_.data(), graph_c_.data(), graph_p_.data(), off.data(),
                                      deps.empty() ? nullptr : deps.data(), &n_ready);
        if (rc != HQS_OK) { last_error_ = hqs_last_error(ctx_); throw std::runtime_error("hqs_graph_push: " + last_error_); }
        if (n_ready != expect_ready)
            std::fprintf(stderr, "[tako_b200] hqs_graph_push: the device and the host mirror disagree on the ready tasks\n");
        graph_h_.clear(); graph_c_.clear(); graph_p_.clear(); graph_deps_.clear();
    }
    if (!forget_h_.empty()) {
        const uint32_t* ready = nullptr;
        uint32_t n_ready = 0;
        if (hqs_graph_finished(ctx_, (uint32_t)forget_h_.size(), forget_h_.data(), &ready, &n_ready) != HQS_OK) {
            last_error_ = hqs_last_error(ctx_);
            std::fprintf(stderr, "[tako_b200] hqs_graph_finished: %s\n", last_error_.c_str());
        }
        for (uint32_t k = 0; k < n_ready; ++k) {
            TaskState& t = tasks_[ready[k]];
            t.waiting = false;
            t.live = true;
        }
        forget_h_.clear();
    }
}

}  // namespace tako_b200

using namespace tako_b200;

// A zero-duration drain on the GPU: seeded random jobs whose tasks depend on tasks of earlier jobs (live, running or
// finished) and on earlier tasks of the same job are submitted between ticks; some waiting tasks are cancelled together with
// their consumers, as tako cancels a job.  Every tick's tasks finish before the next tick.  Checks: every task that is not
// cancelled runs exactly once, never before a dependency that was live at its submit has finished, the worker's free vector
// returns to its total, and the host mirror ends with nothing waiting.
extern "C" int hqshim_selftest_graph(int device, int verbose) {
    int failed = 0;
    auto check = [&](bool ok, const char* what) {
        if (!ok) { ++failed; std::fprintf(stderr, "[shim graph selftest] FAILED: %s\n", what); }
        else if (verbose) std::fprintf(stderr, "[shim graph selftest] ok: %s\n", what);
    };
    try {
        GpuCore core(1, device);
        std::vector<ResourceRqId> rqs;
        for (uint64_t c = 1; c <= 3; ++c) {
            ResourceRequest rq;
            rq.entries.push_back({0, false, c * FRACTIONS_PER_UNIT});
            rqs.push_back(core.get_or_create_resource_rq_id(ResourceRequestVariants{{rq}}));
        }
        core.on_new_worker(50, {24 * FRACTIONS_PER_UNIT});
        core.on_new_worker(51, {16 * FRACTIONS_PER_UNIT});
        uint64_t x = 0x9E3779B97F4A7C15ull;
        auto rnd = [&](uint64_t n) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x % n; };
        enum { WAITING, RUNNING, DONE, CANCELLED };
        std::map<uint64_t, int> state;                          // TaskId -> state
        std::map<uint64_t, std::vector<uint64_t>> live_deps;    // the dependencies that were not finished at submit
        std::map<uint64_t, std::vector<uint64_t>> consumers;
        std::vector<uint64_t> all;
        bool order_ok = true, once_ok = true;
        size_t submitted = 0, ran = 0, cancelled = 0;
        uint32_t job = 1;
        for (int tick = 0; tick < 400; ++tick) {
            if (tick < 120 && rnd(2) == 0) {                    // a new job
                const uint32_t k = 1 + (uint32_t)rnd(30);
                std::vector<NewTask> batch;
                for (uint32_t t = 1; t <= k; ++t) {
                    NewTask nt{TaskId{job, t}, rqs[rnd(rqs.size())], priority_from_user((int32_t)rnd(3)), {}};
                    const uint32_t nd = (uint32_t)rnd(4);
                    for (uint32_t j = 0; j < nd; ++j) {
                        TaskId d;
                        if (rnd(2) == 0 && t > 1) d = TaskId{job, 1 + (uint32_t)rnd(t - 1)};
                        else if (!all.empty()) { const uint64_t v = all[all.size() - 1 - rnd(std::min<size_t>(all.size(), 200))]; d = TaskId{(uint32_t)(v >> 32), (uint32_t)v}; }
                        else continue;
                        bool dup = false;
                        for (const TaskId& e : nt.deps) dup |= e == d;
                        if (!dup) nt.deps.push_back(d);
                    }
                    const uint64_t me = nt.id.as_u64();
                    for (const TaskId& d : nt.deps) {
                        auto s = state.find(d.as_u64());
                        if (s != state.end() && (s->second == WAITING || s->second == RUNNING)) {
                            live_deps[me].push_back(d.as_u64());
                            consumers[d.as_u64()].push_back(me);
                        }
                    }
                    state[me] = WAITING;
                    batch.push_back(nt);
                }
                for (const NewTask& nt : batch) all.push_back(nt.id.as_u64());
                submitted += k;
                core.on_new_tasks(batch);
                ++job;
            }
            if (tick % 7 == 3 && !all.empty()) {               // cancel a waiting task and, transitively, its waiting consumers
                const uint64_t v = all[rnd(all.size())];
                std::vector<uint64_t> stack{v};
                while (!stack.empty()) {
                    const uint64_t c = stack.back();
                    stack.pop_back();
                    if (state[c] != WAITING) continue;
                    state[c] = CANCELLED;
                    ++cancelled;
                    core.remove_ready_task(TaskId{(uint32_t)(c >> 32), (uint32_t)c});
                    for (uint64_t n : consumers[c]) stack.push_back(n);
                }
            }
            const WorkerTaskMapping m = core.run_scheduling();
            std::vector<uint64_t> now;
            for (const auto& kv : m.workers)
                for (const auto& tv : kv.second.assigned) now.push_back(tv.first.as_u64());
            for (uint64_t t : now) {
                once_ok &= state[t] == WAITING;
                for (uint64_t d : live_deps[t]) order_ok &= state[d] == DONE;
                state[t] = RUNNING;
            }
            for (uint64_t t : now) {
                state[t] = DONE;
                ++ran;
                core.on_task_finished(TaskId{(uint32_t)(t >> 32), (uint32_t)t});
            }
            if (tick >= 120 && now.empty() && ran + cancelled == submitted) break;
        }
        check(once_ok, "no task runs twice or after it was cancelled");
        check(order_ok, "no task runs before a dependency that was live at its submit");
        check(ran + cancelled == submitted, "every task that was not cancelled ran");
        check(core.n_waiting() == 0, "nothing waits at the end");
        check(core.free_resources(50)[0] == 24 * FRACTIONS_PER_UNIT && core.free_resources(51)[0] == 16 * FRACTIONS_PER_UNIT,
              "the workers' resources are all back");
        if (verbose) std::fprintf(stderr, "[shim graph selftest] %zu tasks, %zu ran, %zu cancelled\n", submitted, ran, cancelled);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "[shim graph selftest] exception: %s\n", e.what());
        ++failed;
    }
    return failed;
}
