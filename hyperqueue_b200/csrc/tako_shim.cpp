// tako_shim.cpp — implementation of include/tako_shim.hpp: the host side of the tick over the C ABI.
// Everything below the calls to hqs_* happens in libhqsched_b200.so (CUDA); this file is plain C++17.
#include "../../include/tako_shim.hpp"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>

namespace tako_b200 {

namespace {
void log_error(const char* what, const char* msg) { std::fprintf(stderr, "[tako_b200] %s: %s\n", what, msg ? msg : "?"); }
}  // namespace

GpuCore::GpuCore(uint32_t n_resources, int device, uint32_t create_flags) : R_(n_resources) {
    const int rc = hqs_create(&ctx_, device, n_resources, create_flags);
    if (rc != HQS_OK) {
        const char* m = hqs_last_error(nullptr);
        throw std::runtime_error(std::string("hqs_create failed: ") + (m ? m : "?"));
    }
}

GpuCore::~GpuCore() {
    if (ctx_) hqs_destroy(ctx_);
}

// ResourceRqMap::get_or_create (map.rs:99-109): identical variant lists share one id; ids are dense and append-only.
ResourceRqId GpuCore::get_or_create_resource_rq_id(const ResourceRequestVariants& rqv) {
    if (rqv.variants.empty() || rqv.variants.size() > HQS_MAX_VARIANTS)
        throw std::invalid_argument("a request needs 1..8 variants");
    hqs_class cls;
    std::memset(&cls, 0, sizeof cls);
    cls.n_variants = (uint32_t)rqv.variants.size();
    for (size_t v = 0; v < rqv.variants.size(); ++v) {
        const ResourceRequest& rq = rqv.variants[v];
        if (rq.n_nodes != 0) throw std::invalid_argument("multi-node requests are outside this path");
        if (rq.entries.empty()) throw std::invalid_argument("empty resource request");     // request.rs:191-194
        hqs_variant& hv = cls.variants[v];
        for (const ResourceAllocRequest& e : rq.entries) {
            if (e.resource_id >= R_) throw std::invalid_argument("resource id out of range");
            if (e.all) hv.all_mask |= 1u << e.resource_id;
            else {
                if (e.amount == 0) throw std::invalid_argument("Zero resources cannot be requested");   // request.rs:24-32
                hv.amount[e.resource_id] = e.amount;
            }
        }
        hv.weight = rq.weight;
        hv.min_time_ms = rq.min_time_ms;
    }
    const std::string key(reinterpret_cast<const char*>(&cls), sizeof cls);
    auto it = rq_ids_.find(key);
    if (it != rq_ids_.end()) return it->second;
    const ResourceRqId id = (ResourceRqId)classes_.size();
    classes_.push_back(cls);
    rq_ids_.emplace(key, id);
    classes_dirty_ = true;
    return id;
}

void GpuCore::flush_classes() {
    if (!classes_dirty_ || classes_.empty()) return;
    if (hqs_classes_set(ctx_, (uint32_t)classes_.size(), classes_.data()) != HQS_OK) {
        last_error_ = hqs_last_error(ctx_);
        throw std::runtime_error("hqs_classes_set: " + last_error_);
    }
    classes_dirty_ = false;
}

void GpuCore::on_new_worker(WorkerId id, const std::vector<ResourceAmount>& resources, float min_utilization,
                            std::optional<uint64_t> termination_ms) {
    if (workers_.count(id)) throw std::invalid_argument("worker id exists");
    if (workers_.size() >= HQS_MAX_WORKERS) throw std::invalid_argument("too many workers");
    WorkerState w;
    w.total.assign(R_, 0);
    for (size_t r = 0; r < resources.size() && r < R_; ++r) w.total[r] = resources[r];
    w.free = w.total;                                   // worker.rs:40-61: a new worker has everything free
    w.min_utilization = min_utilization;
    w.termination_ms = termination_ms;
    workers_.emplace(id, std::move(w));
}

void GpuCore::on_remove_worker(WorkerId id) {
    auto it = workers_.find(id);
    if (it == workers_.end()) return;
    workers_.erase(it);
    // its running tasks return to the ready queues (reactor.rs:104-150)
    for (uint32_t h = 0; h < tasks_.size(); ++h) {
        TaskState& t = tasks_[h];
        if (t.live && t.worker == (int64_t)id) {
            t.worker = -1;
            push_h_.push_back(h); push_c_.push_back(t.rq); push_p_.push_back(t.priority);
        }
    }
}

void GpuCore::block_request(WorkerId id, ResourceRqId rq, ResourceVariantId v) {
    auto it = workers_.find(id);
    if (it == workers_.end()) return;
    auto& b = it->second.blocked;
    if (std::find(b.begin(), b.end(), std::make_pair(rq, v)) == b.end()) b.emplace_back(rq, v);
}

void GpuCore::unblock_request(WorkerId id, ResourceRqId rq, ResourceVariantId v) {
    auto it = workers_.find(id);
    if (it == workers_.end()) return;
    auto& b = it->second.blocked;
    b.erase(std::remove(b.begin(), b.end(), std::make_pair(rq, v)), b.end());
}

// on_new_tasks (reactor.rs:188-220): the tasks of a submit become known.  Handles are given out here in ascending
// TaskId — the device pops a (priority, class) group in ascending handle, the reference in ascending TaskId
// (taskqueue.rs:395-420) — and job ids grow with every submit, so handle order == TaskId order across submits too.
void GpuCore::on_new_tasks(std::vector<TaskId> tasks) {
    std::sort(tasks.begin(), tasks.end(), [](const TaskId& a, const TaskId& b) { return a.as_u64() < b.as_u64(); });
    for (const TaskId& t : tasks) handle_of(t);
}

size_t GpuCore::n_waiting() const {
    size_t n = 0;
    for (const TaskState& t : tasks_) n += t.waiting ? 1 : 0;
    return n;
}

// A task that was never announced through on_new_tasks gets its handle on first use (arrival order).
uint32_t GpuCore::handle_of(TaskId task) {
    auto it = handle_of_.find(task.as_u64());
    if (it != handle_of_.end()) return it->second;
    if (tasks_.size() >= handle_end_)       // handle 0xFFFFFFFF is reserved: a wrap would alias a live task's handle
        throw std::length_error("the task handle space is exhausted: retire the handles of forgotten tasks (retire_handles)");
    const uint32_t h = (uint32_t)tasks_.size();
    tasks_.emplace_back();
    tasks_[h].id = task;
    handle_of_.emplace(task.as_u64(), h);
    return h;
}

void GpuCore::add_ready_task(TaskId task, ResourceRqId rq, Priority priority) {
    if (rq >= classes_.size()) throw std::invalid_argument("unknown resource request id");
    const uint32_t h = handle_of(task);
    TaskState& t = tasks_[h];
    t.rq = rq; t.priority = priority; t.worker = -1; t.live = true;
    push_h_.push_back(h); push_c_.push_back(rq); push_p_.push_back(priority);     // batched until the next tick
}

void GpuCore::remove_ready_task(TaskId task) {
    auto it = handle_of_.find(task.as_u64());
    if (it == handle_of_.end()) return;
    const uint32_t h = it->second;
    tasks_[h].live = false;
    tasks_[h].waiting = false;
    // still in the host-side batch?
    for (size_t i = 0; i < push_h_.size(); ++i)
        if (push_h_[i] == h) {
            push_h_.erase(push_h_.begin() + i); push_c_.erase(push_c_.begin() + i); push_p_.erase(push_p_.begin() + i);
            return;
        }
    for (size_t i = 0; i < graph_h_.size(); ++i)
        if (graph_h_[i] == h) {
            graph_h_.erase(graph_h_.begin() + i); graph_c_.erase(graph_c_.begin() + i); graph_p_.erase(graph_p_.begin() + i);
            graph_deps_.erase(graph_deps_.begin() + i);
            return;
        }
    if (hqs_ready_remove(ctx_, 1, &h) != HQS_OK) { last_error_ = hqs_last_error(ctx_); log_error("hqs_ready_remove", last_error_.c_str()); }
}

void GpuCore::flush_ready() {
    if (graph_flush_) {                     // the core has submitted tasks with dependencies (tako_shim_graph.cpp)
        (this->*graph_flush_)();
        return;
    }
    if (!forget_h_.empty()) {
        // finished tasks leave the device table for good, so their handles stop pinning priority levels (the device
        // prunes levels without tasks: tako priorities carry a per-job component)
        if (hqs_ready_remove(ctx_, (uint32_t)forget_h_.size(), forget_h_.data()) != HQS_OK) {
            last_error_ = hqs_last_error(ctx_); log_error("hqs_ready_remove (finished tasks)", last_error_.c_str());
        }
        forget_h_.clear();
    }
    if (push_h_.empty()) return;
    flush_classes();
    const int rc = hqs_ready_push(ctx_, (uint32_t)push_h_.size(), push_h_.data(), push_c_.data(), push_p_.data());
    if (rc != HQS_OK) { last_error_ = hqs_last_error(ctx_); throw std::runtime_error("hqs_ready_push: " + last_error_); }
    push_h_.clear(); push_c_.clear(); push_p_.clear();
}

const std::vector<ResourceAmount>& GpuCore::free_resources(WorkerId id) const {
    auto it = workers_.find(id);
    if (it == workers_.end()) throw std::invalid_argument("unknown worker");
    return it->second.free;
}

hqs_stats GpuCore::stats() const {
    hqs_stats st;
    std::memset(&st, 0, sizeof st);
    hqs_get_stats(ctx_, &st);
    return st;
}

// The per-tick worker view of run_scheduling_inner (main.rs:40-46) in the form the C ABI takes: pending classes and ready
// tasks are flushed, the workers come in ascending id, the record buffer is sized, the prefill mask is handed over.
// Returns false when there is nothing to schedule.
bool GpuCore::tick_input(uint64_t now_ms, TickInput& in) {
    flush_classes();
    flush_ready();
    const uint32_t W = (uint32_t)workers_.size();
    if (W == 0 || classes_.empty() || tasks_.empty()) return false;
    const uint32_t Q = (uint32_t)classes_.size();
    std::vector<hqs_worker>& hw = in.hw;
    std::vector<uint64_t>&free_rw = in.free_rw, &total_rw = in.total_rw;
    std::vector<uint8_t>& blocked = in.blocked;
    std::vector<WorkerId>& ids = in.ids;
    hw.assign(W, hqs_worker{});
    free_rw.assign((size_t)W * R_, 0); total_rw.assign((size_t)W * R_, 0); in.free_after.assign((size_t)W * R_, 0);
    ids.assign(W, 0);
    uint32_t i = 0;
    bool any_blocked = false;
    for (const auto& kv : workers_) any_blocked |= !kv.second.blocked.empty();
    blocked.clear();
    if (any_blocked) blocked.assign((size_t)W * Q, 0);
    for (const auto& kv : workers_) {                      // ascending id (solver.rs:44)
        const WorkerState& w = kv.second;
        ids[i] = kv.first;
        std::memset(&hw[i], 0, sizeof(hqs_worker));
        hw[i].worker_id = kv.first;
        hw[i].remaining_time_ms = !w.termination_ms ? HQS_TIME_INF : (*w.termination_ms > now_ms ? *w.termination_ms - now_ms : 0);
        hw[i].min_utilization = w.min_utilization;
        std::copy(w.free.begin(), w.free.end(), free_rw.begin() + (size_t)i * R_);
        std::copy(w.total.begin(), w.total.end(), total_rw.begin() + (size_t)i * R_);
        for (const auto& b : w.blocked)
            if (b.first < Q) blocked[(size_t)i * Q + b.first] |= (uint8_t)(1u << b.second);
        ++i;
    }
    if (out_.size() < tasks_.size() * (pf_max_ ? 2 : 1)) out_.resize(tasks_.size() * (pf_max_ ? 2 : 1));
    if (pf_max_) {
        // Worker::prefilled_tasks as the device needs it: does worker w hold a prefilled task of class c?
        std::vector<uint8_t> pfwc((size_t)W * Q, 0);
        for (const TaskState& t : tasks_)
            if (t.live && t.prefilled_on >= 0) {
                auto it = std::lower_bound(ids.begin(), ids.end(), (WorkerId)t.prefilled_on);
                if (it != ids.end() && *it == (WorkerId)t.prefilled_on) pfwc[(size_t)(it - ids.begin()) * Q + t.rq] = 1;
            }
        hqs_prefill_state(ctx_, W, pfwc.data());
    }
    return true;
}

// the free vectors after the tick replace the host mirror's
void GpuCore::apply_free_after(const TickInput& in) {
    uint32_t i = 0;
    for (auto& kv : workers_) {
        std::copy(in.free_after.begin() + (size_t)i * R_, in.free_after.begin() + (size_t)(i + 1) * R_, kv.second.free.begin());
        ++i;
    }
}

// run_scheduling_inner (main.rs:40-46): builds the per-tick worker view, runs the tick, applies the result to the
// host mirror (Worker::insert_sn_task: free -= request; task state Waiting -> Assigned) and groups it per worker.
WorkerTaskMapping GpuCore::run_scheduling(uint64_t now_ms) {
    WorkerTaskMapping mapping;
    TickInput in;
    if (!tick_input(now_ms, in)) return mapping;
    const uint32_t W = (uint32_t)in.hw.size();
    const std::vector<WorkerId>& ids = in.ids;
    uint32_t n = 0;
    const int rc = hqs_tick(ctx_, W, in.hw.data(), in.free_rw.data(), in.total_rw.data(), in.blocked.empty() ? nullptr : in.blocked.data(),
                            (uint32_t)out_.size(), out_.data(), &n, in.free_after.data());
    if (rc != HQS_OK) {                                    // the reference logs and schedules nothing (solver.rs:412-415)
        last_error_ = hqs_last_error(ctx_);
        log_error("tick failed, nothing scheduled", last_error_.c_str());
        return mapping;
    }
    // min_utilization (solver.rs:154-156, 479-518) is enforced inside the tick: a worker that would receive less than its
    // minimum is taken out of the solve, which then starts over, so nothing has to be handed back here
    for (uint32_t k = 0; k < n; ++k) {
        const hqs_assignment& a = out_[k];
        TaskState& t = tasks_[a.task];
        if (a.kind == 1) {                                  // prefill: the task stays ready (mapping.rs:156-230)
            t.prefilled_on = ids[a.worker];
            mapping.workers[ids[a.worker]].prefills.push_back(t.id);
            continue;
        }
        if (a.kind == 2) {                                  // was prefilled elsewhere: retract + redirect (mapping.rs:63-101)
            mapping.workers[(WorkerId)t.prefilled_on].retracts.push_back(t.id);
            redirects_[t.id.as_u64()] = {ids[a.worker], a.variant};
            t.retracting_from = t.prefilled_on;
            t.prefilled_on = -1;
            t.worker = ids[a.worker];                       // the target's resources are taken already (free_after)
            t.variant = a.variant;
            continue;
        }
        t.worker = ids[a.worker];
        t.variant = a.variant;
        mapping.workers[ids[a.worker]].assigned.emplace_back(t.id, a.variant);     // emission order = priority desc
    }
    apply_free_after(in);
    return mapping;
}

void GpuCore::set_scheduler_config(uint32_t proactive_filling_reserve, uint32_t proactive_filling_max) {
    pf_max_ = proactive_filling_max;
    if (hqs_prefill_config(ctx_, proactive_filling_reserve, proactive_filling_max) != HQS_OK) {
        last_error_ = hqs_last_error(ctx_);
        throw std::runtime_error("hqs_prefill_config: " + last_error_);
    }
}

size_t GpuCore::n_prefilled(WorkerId id) const {
    size_t n = 0;
    for (const TaskState& t : tasks_) n += (t.live && t.prefilled_on == (int64_t)id) ? 1 : 0;
    return n;
}

void GpuCore::on_task_running_prefilled(TaskId task, ResourceVariantId variant) {
    auto it = handle_of_.find(task.as_u64());
    if (it == handle_of_.end()) return;
    TaskState& t = tasks_[it->second];
    if (t.prefilled_on < 0) return;
    auto wit = workers_.find((WorkerId)t.prefilled_on);
    if (wit != workers_.end()) {
        const hqs_variant& hv = classes_[t.rq].variants[variant];
        for (uint32_t r = 0; r < R_; ++r) {                   // Worker::insert_sn_task (worker.rs:188-196)
            if ((hv.all_mask >> r) & 1) wit->second.free[r] = 0;
            else if (hv.amount[r] && wit->second.free[r] != HQS_AMOUNT_MAX) wit->second.free[r] -= std::min(wit->second.free[r], hv.amount[r]);
        }
    }
    t.worker = t.prefilled_on; t.variant = variant; t.prefilled_on = -1;
    const uint32_t h = it->second;
    if (hqs_ready_remove(ctx_, 1, &h) != HQS_OK) { last_error_ = hqs_last_error(ctx_); log_error("hqs_ready_remove", last_error_.c_str()); }
}

std::map<WorkerId, std::vector<std::pair<TaskId, ResourceVariantId>>> GpuCore::on_retract_response(WorkerId worker, const std::vector<TaskId>& tasks) {
    std::map<WorkerId, std::vector<std::pair<TaskId, ResourceVariantId>>> to_workers;
    for (const TaskId& id : tasks) {
        auto it = handle_of_.find(id.as_u64());
        if (it == handle_of_.end()) continue;
        TaskState& t = tasks_[it->second];
        if (t.retracting_from != (int64_t)worker) continue;             // "Retracted task is in invalid state"
        t.retracting_from = -1;
        auto rd = redirects_.find(id.as_u64());
        if (rd != redirects_.end()) {
            to_workers[rd->second.first].emplace_back(id, rd->second.second);
            redirects_.erase(rd);
        }
    }
    return to_workers;
}

// task_finished (reactor.rs:500-580) -> Worker::remove_sn_task -> WorkerResources::add (workerload.rs:194-202):
// free += amount, `All` => free = total.
void GpuCore::on_task_finished(TaskId task) {
    auto it = handle_of_.find(task.as_u64());
    if (it == handle_of_.end()) return;
    TaskState& t = tasks_[it->second];
    if (!t.live || t.worker < 0) return;
    auto wit = workers_.find((WorkerId)t.worker);
    if (wit != workers_.end()) {
        WorkerState& w = wit->second;
        const hqs_variant& hv = classes_[t.rq].variants[t.variant];
        for (uint32_t r = 0; r < R_; ++r) {
            if ((hv.all_mask >> r) & 1) w.free[r] = w.total[r];
            else if (hv.amount[r] && w.free[r] != HQS_AMOUNT_MAX) w.free[r] += hv.amount[r];
        }
    }
    t.worker = -1;
    t.live = false;
    t.forgotten = true;
    forget_h_.push_back(it->second);
}

}  // namespace tako_b200

// =================================================================================================
// self-test
// =================================================================================================
namespace {
using namespace tako_b200;

struct Checker {
    int failed = 0, verbose = 0;
    void check(bool ok, const char* what) {
        if (!ok) { ++failed; std::fprintf(stderr, "[shim selftest] FAILED: %s\n", what); }
        else if (verbose) std::fprintf(stderr, "[shim selftest] ok: %s\n", what);
    }
};

ResourceRequestVariants cpus(uint64_t n, uint64_t gpus_fractions = 0) {
    ResourceRequest rq;
    rq.entries.push_back({0, false, n * FRACTIONS_PER_UNIT});
    if (gpus_fractions) rq.entries.push_back({1, false, gpus_fractions});
    return ResourceRequestVariants{{rq}};
}

// how many tasks of each request id every worker got
std::map<WorkerId, std::map<ResourceRqId, int>> counts(const WorkerTaskMapping& m, const std::map<uint64_t, ResourceRqId>& rq_of) {
    std::map<WorkerId, std::map<ResourceRqId, int>> out;
    for (const auto& kv : m.workers)
        for (const auto& tv : kv.second.assigned) out[kv.first][rq_of.at(tv.first.as_u64())]++;
    return out;
}
}  // namespace

extern "C" int hqshim_selftest(int device, int verbose) {
    Checker ck;
    ck.verbose = verbose;
    try {
        {   // restated from test_schedule_multiple_resources2 (test_scheduler_sn.rs:676-721): workers (6 cpus, 2 gpus) and
            // (6 cpus, 0 gpus); ten 2-cpu tasks and ten (2 cpus + 1 gpu) tasks => [gpu, gpu, plain] and [plain x3]
            GpuCore core(2, device);
            const ResourceRqId plain = core.get_or_create_resource_rq_id(cpus(2));
            const ResourceRqId gpu = core.get_or_create_resource_rq_id(cpus(2, 1 * FRACTIONS_PER_UNIT));
            ck.check(core.get_or_create_resource_rq_id(cpus(2)) == plain, "identical requests are interned");
            core.on_new_worker(50, {6 * FRACTIONS_PER_UNIT, 2 * FRACTIONS_PER_UNIT});
            core.on_new_worker(51, {6 * FRACTIONS_PER_UNIT, 0});
            std::map<uint64_t, ResourceRqId> rq_of;
            for (uint32_t t = 1; t <= 20; ++t) {
                const ResourceRqId rq = t <= 10 ? plain : gpu;
                core.add_ready_task(TaskId{1, t}, rq, priority_from_user(0));
                rq_of[TaskId{1, t}.as_u64()] = rq;
            }
            const WorkerTaskMapping m = core.run_scheduling();
            auto c = counts(m, rq_of);
            ck.check(m.n_assigned() == 6, "multiple resources: six tasks placed");
            ck.check(c[50][gpu] == 2 && c[50][plain] == 1, "worker with gpus: two gpu tasks and one plain");
            ck.check(c[51][plain] == 3 && c[51][gpu] == 0, "worker without gpus: three plain tasks");
            ck.check(core.free_resources(50)[0] == 0 && core.free_resources(50)[1] == 0, "free vector follows the placements");
            // finish one gpu task on worker 50: its resources return and the next tick places another gpu task there
            TaskId done{};
            for (const auto& tv : m.workers.at(50).assigned)
                if (rq_of[tv.first.as_u64()] == gpu) done = tv.first;
            core.on_task_finished(done);
            ck.check(core.free_resources(50)[0] == 2 * FRACTIONS_PER_UNIT && core.free_resources(50)[1] == 1 * FRACTIONS_PER_UNIT,
                     "task_finished returns the resources");
            const WorkerTaskMapping m2 = core.run_scheduling();
            ck.check(m2.n_assigned() == 1 && m2.workers.count(50) == 1 && rq_of[m2.workers.at(50).assigned[0].first.as_u64()] == gpu,
                     "second tick refills the freed slot with the gpu class");
        }
        {   // restated from test_schedule_priorities (test_scheduler_sn.rs:150-307): one 4-cpu worker; priorities 9 (2 cpus),
            // 7 (1 cpu), 6 (2 cpus) => the 2-cpu@9 and the 1-cpu@7 run, the per-worker list is priority-descending
            GpuCore core(1, device);
            const ResourceRqId c2 = core.get_or_create_resource_rq_id(cpus(2)), c1 = core.get_or_create_resource_rq_id(cpus(1));
            core.on_new_worker(50, {4 * FRACTIONS_PER_UNIT});
            core.add_ready_task(TaskId{1, 1}, c2, priority_from_user(9));
            core.add_ready_task(TaskId{1, 2}, c1, priority_from_user(7));
            core.add_ready_task(TaskId{1, 3}, c2, priority_from_user(6));
            const WorkerTaskMapping m = core.run_scheduling();
            ck.check(m.n_assigned() == 2, "priorities: two tasks fit");
            const auto& a = m.workers.at(50).assigned;
            ck.check(a.size() == 2 && a[0].first == TaskId{1, 1} && a[1].first == TaskId{1, 2}, "priority-descending per-worker order");
        }
        {   // blocked request + time limit (worker.rs:320-344): the blocked worker gets nothing of that class; a task with
            // min_time beyond the worker's remaining lifetime is not placed there
            GpuCore core(1, device);
            ResourceRequestVariants longrq = cpus(1);
            longrq.variants[0].min_time_ms = 60000;
            const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1)), cl = core.get_or_create_resource_rq_id(longrq);
            core.on_new_worker(50, {2 * FRACTIONS_PER_UNIT});
            core.on_new_worker(51, {2 * FRACTIONS_PER_UNIT}, 0.0f, 30000);     // terminates in 30 s
            core.block_request(50, c1, 0);
            std::map<uint64_t, ResourceRqId> rq_of;
            for (uint32_t t = 1; t <= 4; ++t) { core.add_ready_task(TaskId{2, t}, c1, priority_from_user(1)); rq_of[TaskId{2, t}.as_u64()] = c1; }
            for (uint32_t t = 5; t <= 8; ++t) { core.add_ready_task(TaskId{2, t}, cl, priority_from_user(0)); rq_of[TaskId{2, t}.as_u64()] = cl; }
            const WorkerTaskMapping m = core.run_scheduling(0);
            auto c = counts(m, rq_of);
            ck.check(c[50][c1] == 0 && c[51][c1] == 2, "blocked request is not placed on the blocking worker");
            ck.check(c[51][cl] == 0 && c[50][cl] == 2, "time request keeps long tasks off the expiring worker");
        }
        {   // zero-duration drain (cfg(zero_worker)): every placement is replayed on the host; nothing may go negative,
            // every task runs exactly once
            GpuCore core(2, device);
            const uint32_t W = 12, N = 5000;
            std::vector<ResourceRqId> rqs;
            for (uint64_t c = 1; c <= 6; ++c) rqs.push_back(core.get_or_create_resource_rq_id(cpus(c, c % 3 ? 0 : 5000)));
            for (uint32_t w = 0; w < W; ++w) core.on_new_worker(100 + w, {32 * FRACTIONS_PER_UNIT, 2 * FRACTIONS_PER_UNIT});
            std::map<uint64_t, ResourceRqId> rq_of;
            uint64_t x = 88172645463325252ull;
            for (uint32_t t = 0; t < N; ++t) {
                x ^= x << 13; x ^= x >> 7; x ^= x << 17;                  // xorshift: seeded synthetic input
                const ResourceRqId rq = rqs[x % rqs.size()];
                core.add_ready_task(TaskId{3, t}, rq, priority_from_user((int32_t)((x >> 20) % 4)));
                rq_of[TaskId{3, t}.as_u64()] = rq;
            }
            std::vector<char> ran(N, 0);
            size_t done = 0, ticks = 0;
            bool ok = true;
            while (done < N && ticks < 10000) {
                const WorkerTaskMapping m = core.run_scheduling();
                if (m.n_assigned() == 0) break;
                for (const auto& kv : m.workers) {
                    uint64_t cpu = 0, gp = 0;
                    for (const auto& tv : kv.second.assigned) {
                        const uint64_t c = rq_of[tv.first.as_u64()] + 1;
                        cpu += c * FRACTIONS_PER_UNIT; gp += (c % 3) ? 0 : 5000;
                        ok &= !ran[tv.first.job_task_id];
                        ran[tv.first.job_task_id] = 1;
                    }
                    ok &= cpu <= 32 * FRACTIONS_PER_UNIT && gp <= 2 * FRACTIONS_PER_UNIT;
                    ok &= core.free_resources(kv.first)[0] == 32 * FRACTIONS_PER_UNIT - cpu;
                }
                for (const auto& kv : m.workers)
                    for (const auto& tv : kv.second.assigned) core.on_task_finished(tv.first);
                done += m.n_assigned();
                ++ticks;
            }
            ck.check(done == N, "drain: every task was scheduled");
            ck.check(ok, "drain: capacities respected, no task twice, free vectors consistent");
            ck.check(ticks > 0 && ticks < 200, "drain: finished in a sane number of ticks");
            if (verbose) std::fprintf(stderr, "[shim selftest] drain took %zu ticks\n", ticks);
        }
        {   // proactive filling + retract / redirect, restated from test_prefill_basic and test_prefill_steal
            // (test_scheduler_sn.rs:1168-1200, 1225-1306)
            GpuCore core(1, device);
            core.set_scheduler_config(4, 32);
            const ResourceRqId c4 = core.get_or_create_resource_rq_id(cpus(4));
            core.on_new_worker(50, {8 * FRACTIONS_PER_UNIT});
            core.on_new_worker(51, {8 * FRACTIONS_PER_UNIT});
            for (uint32_t t = 1; t <= 300; ++t) core.add_ready_task(TaskId{4, t}, c4, priority_from_user(0));
            WorkerTaskMapping m = core.run_scheduling();
            bool ok = m.workers.size() == 2;
            for (const auto& kv : m.workers) ok &= kv.second.prefills.size() == 32 && kv.second.assigned.size() == 2 && kv.second.retracts.empty();
            ck.check(ok, "prefill: 32 prefills + 2 assigned per worker");
            ck.check(core.n_prefilled(50) == 32 && core.n_prefilled(51) == 32, "prefill: Worker::prefilled_tasks mirror");
        }
        {
            GpuCore core(1, device);
            core.set_scheduler_config(3, 6);
            const ResourceRqId c1 = core.get_or_create_resource_rq_id(cpus(1));
            core.on_new_worker(50, {1 * FRACTIONS_PER_UNIT});
            for (uint32_t t = 1; t <= 9; ++t) core.add_ready_task(TaskId{5, t}, c1, priority_from_user(0));
            WorkerTaskMapping m = core.run_scheduling();
            ck.check(core.n_prefilled(50) == 5, "steal: 5 prefills on the only worker");
            core.on_new_worker(51, {5 * FRACTIONS_PER_UNIT});
            m = core.run_scheduling();
            ck.check(m.workers[50].retracts.size() == 2 && m.workers[51].assigned.size() == 3, "steal: 2 retracts, 3 fresh tasks");
            ck.check(core.redirects().size() == 2 && core.n_prefilled(50) == 3 && core.free_resources(51)[0] == 0, "steal: redirects and resources");
            const TaskId t = m.workers[50].retracts[0];
            auto sent = core.on_retract_response(50, {t});
            ck.check(sent.size() == 1 && sent[51].size() == 1 && sent[51][0].first == t && core.redirects().size() == 1, "steal: retract response sends the task on");
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "[shim selftest] exception: %s\n", e.what());
        ++ck.failed;
    }
    return ck.failed;
}
