// tako_shim_grouped.cpp — the part of include/tako_shim.hpp that fetches a tick grouped per worker (hqs_tick_grouped):
// GpuCore::run_scheduling_grouped, its self-test and the timing aid of tools/grouped_probe.py.  Plain C++17 above the C ABI.
#include "../../include/tako_shim.hpp"

#include <chrono>
#include <cstdio>

namespace tako_b200 {

WorkerTaskMapping GpuCore::run_scheduling_grouped(uint64_t now_ms) {
    WorkerTaskMapping mapping;
    TickInput in;
    if (!tick_input(now_ms, in)) return mapping;
    const uint32_t W = (uint32_t)in.hw.size();
    const std::vector<WorkerId>& ids = in.ids;
    // worker w's prefills, then its assignments, each a contiguous run in emission order = priority descending
    uint32_t n = 0;
    std::vector<uint32_t> off(2 * (size_t)W + 2);
    const int rc = hqs_tick_grouped(ctx_, W, in.hw.data(), in.free_rw.data(), in.total_rw.data(), in.blocked.empty() ? nullptr : in.blocked.data(),
                                    (uint32_t)out_.size(), out_.data(), &n, (uint32_t)off.size(), off.data(), in.free_after.data());
    if (rc != HQS_OK) {                                    // the reference logs and schedules nothing (solver.rs:412-415)
        last_error_ = hqs_last_error(ctx_);
        std::fprintf(stderr, "[tako_b200] tick failed, nothing scheduled: %s\n", last_error_.c_str());
        return mapping;
    }
    for (uint32_t w = 0; w < W; ++w) {
        const uint32_t p0 = off[2 * w], a0 = off[2 * w + 1], a1 = off[2 * w + 2];
        if (a1 == p0) continue;
        WorkerTaskUpdate& up = mapping.workers[ids[w]];
        up.prefills.reserve(a0 - p0);
        for (uint32_t k = p0; k < a0; ++k) {                // prefill: the task stays ready (mapping.rs:156-230)
            TaskState& t = tasks_[out_[k].task];
            t.prefilled_on = ids[w];
            up.prefills.push_back(t.id);
        }
        up.assigned.reserve(a1 - a0);
        for (uint32_t k = a0; k < a1; ++k) {
            TaskState& t = tasks_[out_[k].task];
            t.worker = ids[w];
            t.variant = out_[k].variant;
            up.assigned.emplace_back(t.id, out_[k].variant);
        }
    }
    for (uint32_t k = off[2 * (size_t)W]; k < n; ++k) {     // was prefilled elsewhere: retract + redirect (mapping.rs:63-101)
        const hqs_assignment& a = out_[k];
        TaskState& t = tasks_[a.task];
        mapping.workers[(WorkerId)t.prefilled_on].retracts.push_back(t.id);
        redirects_[t.id.as_u64()] = {ids[a.worker], a.variant};
        t.retracting_from = t.prefilled_on;
        t.prefilled_on = -1;
        t.worker = ids[a.worker];                           // the target's resources are taken already (free_after)
        t.variant = a.variant;
    }
    apply_free_after(in);
    return mapping;
}

}  // namespace tako_b200

namespace {
using namespace tako_b200;

bool same_mapping(const WorkerTaskMapping& a, const WorkerTaskMapping& b) {
    if (a.workers.size() != b.workers.size()) return false;
    auto ia = a.workers.begin();
    auto ib = b.workers.begin();
    for (; ia != a.workers.end(); ++ia, ++ib)
        if (ia->first != ib->first || !(ia->second.assigned == ib->second.assigned) || !(ia->second.prefills == ib->second.prefills) ||
            !(ia->second.retracts == ib->second.retracts))
            return false;
    return true;
}

ResourceRequestVariants cpus_rq(uint64_t n) {
    ResourceRequest rq;
    rq.entries.push_back({0, false, n * FRACTIONS_PER_UNIT});
    return ResourceRequestVariants{{rq}};
}
}  // namespace

extern "C" int hqshim_selftest_grouped(int device, int verbose) {
    int failed = 0;
    auto check = [&](bool ok, const char* what) {
        if (!ok) { ++failed; std::fprintf(stderr, "[shim grouped selftest] FAILED: %s\n", what); }
        else if (verbose) std::fprintf(stderr, "[shim grouped selftest] ok: %s\n", what);
    };
    try {
        {   // drain: 6 classes, 4 priorities, 12 workers; every tick's mapping and free vectors must agree
            GpuCore flat(1, device), grouped(1, device);
            GpuCore* cores[2] = {&flat, &grouped};
            const uint32_t W = 12, N = 5000;
            for (GpuCore* c : cores) {
                std::vector<ResourceRqId> rqs;
                for (uint64_t k = 1; k <= 6; ++k) rqs.push_back(c->get_or_create_resource_rq_id(cpus_rq(k)));
                for (uint32_t w = 0; w < W; ++w) c->on_new_worker(100 + w, {32 * FRACTIONS_PER_UNIT});
                uint64_t x = 88172645463325252ull;
                for (uint32_t t = 0; t < N; ++t) {
                    x ^= x << 13; x ^= x >> 7; x ^= x << 17;              // xorshift: seeded synthetic input
                    c->add_ready_task(TaskId{3, t}, rqs[x % rqs.size()], priority_from_user((int32_t)((x >> 20) % 4)));
                }
            }
            bool same = true, frees = true;
            size_t done = 0, ticks = 0;
            while (done < N && ticks < 1000) {
                const WorkerTaskMapping mf = flat.run_scheduling(), mg = grouped.run_scheduling_grouped();
                same &= same_mapping(mf, mg);
                for (uint32_t w = 0; w < W; ++w) frees &= flat.free_resources(100 + w) == grouped.free_resources(100 + w);
                if (mf.n_assigned() == 0) break;
                for (const auto& kv : mf.workers)
                    for (const auto& tv : kv.second.assigned) { flat.on_task_finished(tv.first); grouped.on_task_finished(tv.first); }
                done += mf.n_assigned();
                ++ticks;
            }
            check(done == N && ticks > 1, "drain: every task was scheduled over several ticks");
            check(same, "drain: grouped mapping == flat mapping on every tick, list order included");
            check(frees, "drain: free vectors agree on every tick");
        }
        {   // proactive filling, then a new worker steals prefilled tasks (test_scheduler_sn.rs:1225-1306)
            GpuCore flat(1, device), grouped(1, device);
            GpuCore* cores[2] = {&flat, &grouped};
            for (GpuCore* c : cores) {
                c->set_scheduler_config(3, 6);
                const ResourceRqId c1 = c->get_or_create_resource_rq_id(cpus_rq(1));
                c->on_new_worker(50, {1 * FRACTIONS_PER_UNIT});
                for (uint32_t t = 1; t <= 9; ++t) c->add_ready_task(TaskId{5, t}, c1, priority_from_user(0));
            }
            WorkerTaskMapping mf = flat.run_scheduling(), mg = grouped.run_scheduling_grouped();
            check(same_mapping(mf, mg) && mg.workers[50].prefills.size() == 5 && grouped.n_prefilled(50) == 5, "prefill: 5 prefills, equal mappings");
            for (GpuCore* c : cores) c->on_new_worker(51, {5 * FRACTIONS_PER_UNIT});
            mf = flat.run_scheduling(); mg = grouped.run_scheduling_grouped();
            check(same_mapping(mf, mg) && mg.workers[50].retracts.size() == 2 && mg.workers[51].assigned.size() == 3, "steal: 2 retracts, 3 fresh tasks, equal mappings");
            check(grouped.redirects() == flat.redirects() && grouped.redirects().size() == 2 && grouped.n_prefilled(50) == 3 &&
                  grouped.free_resources(51)[0] == 0, "steal: redirects, prefill mirror and resources");
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "[shim grouped selftest] exception: %s\n", e.what());
        ++failed;
    }
    return failed;
}

extern "C" int hqshim_time_mapping(hqs_ctx* ctx, uint32_t n_workers, const hqs_worker* workers, const uint64_t* free_rw,
                                   const uint64_t* total_rw, uint32_t out_cap, int grouped, uint32_t reps, double* out_ms,
                                   uint64_t* digest) {
    const uint32_t W = n_workers;
    std::vector<hqs_assignment> out(out_cap);
    std::vector<uint32_t> off(2 * (size_t)W + 2);
    for (uint32_t rep = 0; rep < reps; ++rep) {
        int rc = hqs_ready_rearm(ctx);
        if (rc == HQS_OK) rc = hqs_sync(ctx);
        if (rc != HQS_OK) return rc;
        WorkerTaskMapping mapping;
        uint32_t n = 0;
        const auto t0 = std::chrono::steady_clock::now();
        if (grouped) {
            rc = hqs_tick_grouped(ctx, W, workers, free_rw, total_rw, nullptr, out_cap, out.data(), &n, (uint32_t)off.size(), off.data(), nullptr);
            if (rc != HQS_OK) return rc;
            for (uint32_t w = 0; w < W; ++w) {
                const uint32_t a0 = off[2 * w + 1], a1 = off[2 * w + 2];
                if (a1 == a0) continue;
                auto& assigned = mapping.workers[workers[w].worker_id].assigned;
                assigned.reserve(a1 - a0);
                for (uint32_t k = a0; k < a1; ++k) assigned.emplace_back(TaskId{1, out[k].task}, out[k].variant);
            }
        } else {
            rc = hqs_tick(ctx, W, workers, free_rw, total_rw, nullptr, out_cap, out.data(), &n, nullptr);
            if (rc != HQS_OK) return rc;
            for (uint32_t k = 0; k < n; ++k)
                if (out[k].kind == 0)
                    mapping.workers[workers[out[k].worker].worker_id].assigned.emplace_back(TaskId{1, out[k].task}, out[k].variant);
        }
        out_ms[rep] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        uint64_t h = n;
        for (const auto& kv : mapping.workers)
            for (const auto& tv : kv.second.assigned) h = h * 1000003ull + tv.first.as_u64() * 8 + tv.second + kv.first;
        if (digest) *digest = h;
    }
    return HQS_OK;
}
