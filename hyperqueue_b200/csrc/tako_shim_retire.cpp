// tako_shim_retire.cpp — GpuCore::retire_handles (include/tako_shim.hpp) and its GPU self-test.  The only caller of
// hqs_handles_compact: tako_shim.cpp itself does not reference it, so a host that never retires links without it.
#include "../../include/tako_shim.hpp"

#include <algorithm>
#include <cstdio>
#include <exception>
#include <map>
#include <set>
#include <stdexcept>
#include <vector>

namespace tako_b200 {

// The device keeps every VALID handle; the host names the others it still knows (announced, removed from the ready set,
// started prefilled, retracting, ...).  Forgotten tasks left the device table when their finish, cancel or failure was
// flushed, so they are exactly the handles that go.  A retracting task keeps its handle even if it is forgotten: its
// retract response still finds it, as on a core that never retires.
// Announced tasks that never reached the device sit past its table (handles >= its n_handles); they are larger than every
// handle the device renumbers, so they follow the survivors in the same order.
size_t GpuCore::retire_handles() {
    flush_classes();
    flush_ready();                       // submits, pushes and finishes reach the device before it renumbers
    const uint32_t n_dev = stats().n_handles;
    auto kept_by_host = [&](const TaskState& t) { return !t.forgotten || t.retracting_from >= 0; };
    std::vector<uint32_t> keep;
    keep.reserve(n_dev);
    for (uint32_t h = 0; h < n_dev && h < tasks_.size(); ++h)
        if (kept_by_host(tasks_[h])) keep.push_back(h);
    const uint32_t* old_of_new = nullptr;
    uint32_t n_kept = 0;
    if (hqs_handles_compact(ctx_, (uint32_t)keep.size(), keep.data(), &old_of_new, &n_kept) != HQS_OK) {
        last_error_ = hqs_last_error(ctx_);
        throw std::runtime_error("hqs_handles_compact: " + last_error_);
    }
    if (n_kept != keep.size())          // a forgotten handle still VALID on the device: the mirror and the table disagree
        std::fprintf(stderr, "[tako_b200] hqs_handles_compact kept %u handles, the host knows %zu\n", n_kept, keep.size());
    std::vector<TaskState> kept;
    kept.reserve(n_kept + (tasks_.size() - std::min<size_t>(n_dev, tasks_.size())));
    for (uint32_t i = 0; i < n_kept; ++i) kept.push_back(tasks_[old_of_new[i]]);
    for (size_t h = n_dev; h < tasks_.size(); ++h)
        if (kept_by_host(tasks_[h])) kept.push_back(tasks_[h]);
    const size_t retired = tasks_.size() - kept.size();
    handle_of_.clear();
    for (uint32_t i = 0; i < kept.size(); ++i) handle_of_.emplace(kept[i].id.as_u64(), i);
    tasks_.swap(kept);
    return retired;
}

}  // namespace tako_b200

using namespace tako_b200;

namespace {

bool same_mapping(const WorkerTaskMapping& a, const WorkerTaskMapping& b) {
    if (a.workers.size() != b.workers.size()) return false;
    for (auto ia = a.workers.begin(), ib = b.workers.begin(); ia != a.workers.end(); ++ia, ++ib) {
        if (ia->first != ib->first) return false;
        const WorkerTaskUpdate &x = ia->second, &y = ib->second;
        if (x.assigned != y.assigned || x.prefills != y.prefills || x.retracts != y.retracts) return false;
    }
    return true;
}

}  // namespace

// Two cores, one retiring its forgotten handles every few ticks and one never, get the same seeded zero-duration drain: jobs
// whose tasks depend on earlier tasks, proactive filling (prefills, retracts and their responses), cancels of tasks in any
// state, failures of assigned tasks.  Every result must be equal, and the retiring core's handle count must stay bounded.
extern "C" int hqshim_selftest_retire(int device, int verbose) {
    int failed = 0;
    auto check = [&](bool ok, const char* what) {
        if (!ok) { ++failed; std::fprintf(stderr, "[shim retire selftest] FAILED: %s\n", what); }
        else if (verbose) std::fprintf(stderr, "[shim retire selftest] ok: %s\n", what);
    };
    try {
        GpuCore a(1, device), b(1, device);               // a retires, b never does
        GpuCore* both[2] = {&a, &b};
        std::vector<ResourceRqId> rqs;
        for (GpuCore* c : both) {
            c->set_scheduler_config(1, 2);
            rqs.clear();
            for (uint64_t k = 1; k <= 3; ++k) {
                ResourceRequest rq;
                rq.entries.push_back({0, false, k * FRACTIONS_PER_UNIT});
                rqs.push_back(c->get_or_create_resource_rq_id(ResourceRequestVariants{{rq}}));
            }
            c->on_new_worker(50, {12 * FRACTIONS_PER_UNIT});
            c->on_new_worker(51, {8 * FRACTIONS_PER_UNIT});
        }
        uint64_t x = 0x9E3779B97F4A7C15ull;
        auto rnd = [&](uint64_t n) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x % n; };
        auto tid = [](uint64_t v) { return TaskId{(uint32_t)(v >> 32), (uint32_t)v}; };
        std::set<uint64_t> known;                          // tasks tako knows: submitted and not finished, cancelled or failed
        std::vector<uint64_t> recent;
        bool maps_ok = true, lists_ok = true, free_ok = true, bound_ok = true, msgs_ok = true;
        size_t retired = 0, retires = 0, max_handles = 0;
        uint32_t job = 1;
        for (int tick = 0; tick < 400; ++tick) {
            if (tick < 300 && rnd(3) != 0) {
                const uint32_t k = 1 + (uint32_t)rnd(25);
                std::vector<NewTask> batch;
                for (uint32_t t = 1; t <= k; ++t) {
                    NewTask nt{TaskId{job, t}, rqs[rnd(rqs.size())], priority_from_user((int32_t)rnd(3)), {}};
                    for (uint32_t j = 0, nd = (uint32_t)rnd(4); j < nd; ++j) {
                        TaskId d;
                        if (rnd(2) == 0 && t > 1) d = TaskId{job, 1 + (uint32_t)rnd(t - 1)};
                        else if (!recent.empty()) d = tid(recent[recent.size() - 1 - rnd(std::min<size_t>(recent.size(), 150))]);
                        else continue;
                        if (std::find(nt.deps.begin(), nt.deps.end(), d) == nt.deps.end()) nt.deps.push_back(d);
                    }
                    batch.push_back(nt);
                }
                for (const NewTask& nt : batch) { recent.push_back(nt.id.as_u64()); known.insert(nt.id.as_u64()); }
                for (GpuCore* c : both) c->on_new_tasks(batch);
                ++job;
            }
            const WorkerTaskMapping m = a.run_scheduling();
            maps_ok &= same_mapping(m, b.run_scheduling());
            std::vector<uint64_t> running;
            std::vector<std::pair<WorkerId, uint64_t>> retracting;
            for (const auto& kv : m.workers) {
                for (const auto& tv : kv.second.assigned) running.push_back(tv.first.as_u64());
                for (const TaskId& t : kv.second.retracts) retracting.push_back({kv.first, t.as_u64()});
            }
            if (!recent.empty() && rnd(4) == 0) {              // a cancel of tasks in any state, known or not
                std::vector<TaskId> named;
                for (int j = 0, k = 1 + (int)rnd(3); j < k; ++j) named.push_back(tid(recent[rnd(recent.size())]));
                if (!running.empty()) named.push_back(tid(running[rnd(running.size())]));
                const CancelledTasks ra = a.on_cancel_tasks(named), rb = b.on_cancel_tasks(named);
                lists_ok &= ra.cancelled == rb.cancelled;
                msgs_ok &= ra.messages == rb.messages;
                for (const TaskId& t : ra.cancelled) known.erase(t.as_u64());
            }
            if (!running.empty() && rnd(4) == 0) {             // a failure of an assigned task
                const TaskId v = tid(running[rnd(running.size())]);
                const std::vector<TaskId> ca = a.on_task_failed(v), cb = b.on_task_failed(v);
                lists_ok &= ca == cb;
                known.erase(v.as_u64());
                for (const TaskId& t : ca) known.erase(t.as_u64());
            }
            for (const auto& wr : retracting) {                // the retracted tasks come back and run on their targets
                const auto sa = a.on_retract_response(wr.first, {tid(wr.second)});
                msgs_ok &= sa == b.on_retract_response(wr.first, {tid(wr.second)});
                for (const auto& kv : sa)
                    for (const auto& tv : kv.second) running.push_back(tv.first.as_u64());
            }
            for (uint64_t v : running) {
                for (GpuCore* c : both) c->on_task_finished(tid(v));
                known.erase(v);
            }
            for (WorkerId w : {50u, 51u}) free_ok &= a.free_resources(w) == b.free_resources(w);
            if (tick % 3 == 2) {
                retired += a.retire_handles();
                ++retires;
                bound_ok &= a.n_handles() <= known.size() + a.redirects().size();
                max_handles = std::max(max_handles, a.n_handles());
            }
            if (tick >= 300 && known.empty()) break;
        }
        check(maps_ok, "every WorkerTaskMapping equals the one of a core that never retires");
        check(lists_ok && msgs_ok, "cancel, failure and retract results equal the ones of a core that never retires");
        check(free_ok, "the free vectors equal the ones of a core that never retires");
        check(bound_ok, "after each retire n_handles is at most the tasks tako still knows");
        check(retired > 0 && a.n_handles() < b.n_handles(), "handles were retired");
        check(a.n_waiting() == b.n_waiting() && a.redirects() == b.redirects(), "waiting tasks and redirects agree");
        if (verbose)
            std::fprintf(stderr, "[shim retire selftest] %zu retires, %zu handles retired, at most %zu handles after a retire "
                         "(%zu without)\n", retires, retired, max_handles, b.n_handles());
        // the end of the handle space
        GpuCore c(1, device);
        c.limit_handles_for_testing(3);
        c.on_new_tasks(std::vector<TaskId>{TaskId{1, 1}, TaskId{1, 2}, TaskId{1, 3}});
        bool threw = false;
        try { c.on_new_tasks(std::vector<TaskId>{TaskId{1, 4}}); } catch (const std::length_error&) { threw = true; }
        check(threw && c.n_handles() == 3, "handle_of throws at the end of the handle space instead of wrapping");
    } catch (const std::exception& e) {
        std::fprintf(stderr, "[shim retire selftest] exception: %s\n", e.what());
        ++failed;
    }
    return failed;
}
