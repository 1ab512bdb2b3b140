// TEST DOUBLE of the C ABI (include/hqsched.h) — test infrastructure, never shipped or loaded by the product.
// It lets the C++ host shim (hyperqueue_b200/csrc/tako_shim.cpp) be exercised on a box without a GPU: ready set,
// classes and ticks are kept in host memory and a tick is a plain priority-ordered first-fit over variant order.
// Only the entry points the shim calls are implemented.  Proactive filling is modelled in its simplest form (enough to
// drive the shim's bookkeeping of kind 1 / kind 2 records): waiting tasks are taken before prefilled ones, an assigned
// prefilled task comes out as kind 2, and after the assignments every class with waiting tasks left hands
// min((waiting - reserve) / eligible, max) of them to each worker that got an assignment of the class in this tick and
// holds no prefilled task of it (mapping.rs:156-230).
#include "../../include/hqsched.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

struct hqs_ctx {
    uint32_t R = 0;
    std::vector<hqs_class> classes;
    struct T { uint32_t cls; uint64_t prio; bool ready; bool prefilled = false; };
    uint32_t pf_reserve = 0, pf_max = 0;
    std::vector<uint8_t> pfwc;                   // [W][Q] mirror given by hqs_prefill_state (per tick)
    uint32_t pf_W = 0;
    std::map<uint32_t, T> tasks;                 // by handle
    hqs_stats stats{};
    std::string err;
    uint32_t pushes = 0, removes = 0;
};

extern "C" {
int hqs_abi_version(void) { return HQS_ABI_VERSION; }
const char* hqs_last_error(const hqs_ctx* ctx) { return ctx ? ctx->err.c_str() : "fake"; }
int hqs_create(hqs_ctx** out, int, uint32_t n_resources, uint32_t) {
    *out = new hqs_ctx();
    (*out)->R = n_resources;
    return HQS_OK;
}
void hqs_destroy(hqs_ctx* ctx) { delete ctx; }
int hqs_classes_set(hqs_ctx* ctx, uint32_t n, const hqs_class* classes) {
    ctx->classes.assign(classes, classes + n);
    return HQS_OK;
}
int hqs_ready_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id, const uint64_t* priority) {
    for (uint32_t i = 0; i < n; ++i) {
        if (class_id[i] >= ctx->classes.size()) { ctx->err = "class id out of range"; return HQS_E_INVALID; }
        ctx->tasks[task[i]] = {class_id[i], priority[i], true, false};
    }
    ctx->pushes += n;
    return HQS_OK;
}
int hqs_ready_remove(hqs_ctx* ctx, uint32_t n, const uint32_t* task) {
    for (uint32_t i = 0; i < n; ++i) {
        auto it = ctx->tasks.find(task[i]);
        if (it != ctx->tasks.end()) it->second.ready = false;
    }
    ctx->removes += n;
    return HQS_OK;
}
int hqs_get_stats(hqs_ctx* ctx, hqs_stats* out) {
    ctx->stats.n_handles = ctx->tasks.empty() ? 0 : ctx->tasks.rbegin()->first + 1;
    ctx->stats.kernel_launches = ctx->pushes;          // the test reads the push counter through this field
    ctx->stats.n_segments = ctx->removes;
    *out = ctx->stats;
    return HQS_OK;
}
int hqs_tick(hqs_ctx* ctx, uint32_t W, const hqs_worker* workers, const uint64_t* free_rw, const uint64_t* total_rw,
             const uint8_t* blocked, uint32_t out_cap, hqs_assignment* out, uint32_t* out_n, uint64_t* free_after) {
    const uint32_t R = ctx->R, Q = (uint32_t)ctx->classes.size();
    for (uint32_t w = 1; w < W; ++w)
        if (workers[w].worker_id <= workers[w - 1].worker_id) { ctx->err = "workers must be sorted"; return HQS_E_INVALID; }
    std::vector<uint64_t> fr(free_rw, free_rw + (size_t)W * R);
    std::vector<std::pair<std::pair<uint64_t, uint32_t>, uint32_t>> order3;   // (priority desc, waiting before prefilled, handle asc)
    for (auto& kv : ctx->tasks)
        if (kv.second.ready) order3.push_back({{~kv.second.prio, kv.second.prefilled ? 1u : 0u}, kv.first});
    std::sort(order3.begin(), order3.end());
    std::vector<std::pair<uint64_t, uint32_t>> order;
    for (auto& o : order3) order.push_back({o.first.first, o.second});
    std::vector<uint8_t> got((size_t)W * Q, 0);            // worker w got an assignment of class c in this tick
    uint32_t n = 0;
    for (auto& po : order) {
        hqs_ctx::T& t = ctx->tasks[po.second];
        const hqs_class& c = ctx->classes[t.cls];
        bool placed = false;
        for (uint32_t w = 0; w < W && !placed; ++w)
            for (uint32_t v = 0; v < c.n_variants && !placed; ++v) {
                const hqs_variant& hv = c.variants[v];
                if (blocked && ((blocked[(size_t)w * Q + t.cls] >> v) & 1)) continue;
                if (workers[w].remaining_time_ms != HQS_TIME_INF && hv.min_time_ms > workers[w].remaining_time_ms) continue;
                bool ok = true;
                for (uint32_t r = 0; r < R; ++r) {
                    if ((hv.all_mask >> r) & 1) ok &= total_rw[(size_t)w * R + r] != 0 && fr[(size_t)w * R + r] == total_rw[(size_t)w * R + r];
                    else ok &= hv.amount[r] <= fr[(size_t)w * R + r];
                }
                if (!ok || n >= out_cap) continue;
                for (uint32_t r = 0; r < R; ++r) {
                    if ((hv.all_mask >> r) & 1) fr[(size_t)w * R + r] = 0;
                    else fr[(size_t)w * R + r] -= hv.amount[r];
                }
                out[n].task = po.second; out[n].worker = (uint16_t)w; out[n].variant = (uint8_t)v; out[n].kind = t.prefilled ? 2 : 0;
                ++n;
                t.ready = false;
                t.prefilled = false;
                got[(size_t)w * Q + t.cls] = 1;
                placed = true;
            }
    }
    if (ctx->pf_max) {
        for (uint32_t c = 0; c < Q; ++c) {
            std::vector<uint32_t> waiting;                  // handle order
            for (auto& kv : ctx->tasks)
                if (kv.second.ready && !kv.second.prefilled && kv.second.cls == c) waiting.push_back(kv.first);
            if (waiting.size() <= ctx->pf_reserve) continue;
            std::vector<uint32_t> eligible;
            for (uint32_t w = 0; w < W; ++w) {
                const bool holds = ctx->pf_W == W && ctx->pfwc[(size_t)w * Q + c];
                if (got[(size_t)w * Q + c] && !holds) eligible.push_back(w);
            }
            if (eligible.empty()) continue;
            const uint32_t per = std::min<uint32_t>((uint32_t)((waiting.size() - ctx->pf_reserve) / eligible.size()), ctx->pf_max);
            size_t next = 0;
            for (uint32_t w : eligible)
                for (uint32_t k = 0; k < per && n < out_cap; ++k) {
                    const uint32_t h = waiting[next++];
                    ctx->tasks[h].prefilled = true;
                    out[n].task = h; out[n].worker = (uint16_t)w; out[n].variant = 255; out[n].kind = 1;
                    ++n;
                }
        }
    }
    ctx->pfwc.clear(); ctx->pf_W = 0;                       // the mirror is per tick
    *out_n = n;
    if (free_after) std::copy(fr.begin(), fr.end(), free_after);
    ctx->stats.n_assigned = n;
    ctx->stats.solver_path = 0;                             // no device solve loop runs in the double
    ctx->stats.ticks++;
    return HQS_OK;
}
int hqs_prefill_config(hqs_ctx* ctx, uint32_t reserve, uint32_t max_per_worker) {
    ctx->pf_reserve = reserve; ctx->pf_max = max_per_worker;
    return HQS_OK;
}
int hqs_prefill_state(hqs_ctx* ctx, uint32_t n_workers, const uint8_t* prefilled_wc) {
    ctx->pf_W = n_workers;
    ctx->pfwc.assign(prefilled_wc, prefilled_wc + (size_t)n_workers * ctx->classes.size());
    return HQS_OK;
}
int hqs_prefill_dispose(hqs_ctx* ctx, uint32_t class_id) {
    for (auto& kv : ctx->tasks)
        if (kv.second.cls == class_id) kv.second.prefilled = false;
    return HQS_OK;
}
}
