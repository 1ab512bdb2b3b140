// TEST DOUBLE of the C ABI's task-graph calls (hqs_graph_push / hqs_graph_finished, include/hqsched.h) — test infrastructure,
// never shipped or loaded by the product.  It is fake_hqsched.cpp (compiled into this translation unit, so that the graph
// calls reach its ready set) plus the graph semantics in host memory: a dependency counts if its task is VALID (pushed and
// neither finished nor removed) or earlier in the batch; a waiting task sits in the ready set as not ready until its last
// counted producer finishes; an edge releases only the incarnation of the consumer it was made for.  hqs_ready_push,
// hqs_ready_remove and hqs_destroy wrap the double's own versions to keep the set of VALID handles and the consumer lists.
#define hqs_ready_push fake_base_ready_push
#define hqs_ready_remove fake_base_ready_remove
#define hqs_destroy fake_base_destroy
#include "fake_hqsched.cpp"
#undef hqs_ready_push
#undef hqs_ready_remove
#undef hqs_destroy

#include <set>

namespace {
struct GraphState {
    std::set<uint32_t> valid;
    std::map<uint32_t, uint32_t> deps, gen;
    std::map<uint32_t, std::vector<std::pair<uint32_t, uint32_t>>> cons;   // producer -> (consumer, incarnation)
    std::vector<uint32_t> new_ready;
};
std::map<const hqs_ctx*, GraphState> g_graph;
}  // namespace

extern "C" {
int hqs_ready_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id, const uint64_t* priority) {
    const int rc = fake_base_ready_push(ctx, n, task, class_id, priority);
    if (rc == HQS_OK)
        for (uint32_t i = 0; i < n; ++i) g_graph[ctx].valid.insert(task[i]);
    return rc;
}
int hqs_ready_remove(hqs_ctx* ctx, uint32_t n, const uint32_t* task) {
    GraphState& g = g_graph[ctx];
    for (uint32_t i = 0; i < n; ++i) {
        g.valid.erase(task[i]);
        g.cons.erase(task[i]);
    }
    return fake_base_ready_remove(ctx, n, task);
}
void hqs_destroy(hqs_ctx* ctx) {
    g_graph.erase(ctx);
    fake_base_destroy(ctx);
}
int hqs_graph_push(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t* class_id, const uint64_t* priority,
                   const uint32_t* dep_off, const uint32_t* deps, uint32_t* n_ready) {
    GraphState& g = g_graph[ctx];
    std::map<uint32_t, uint32_t> pos;
    for (uint32_t i = 0; i < n; ++i) {
        if (class_id[i] >= ctx->classes.size()) { ctx->err = "class id out of range"; return HQS_E_INVALID; }
        if (g.valid.count(task[i]) || !pos.emplace(task[i], i).second) { ctx->err = "live or repeated handle"; return HQS_E_INVALID; }
    }
    uint32_t made = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t h = task[i], k = ++g.gen[h];
        uint32_t cnt = 0;
        for (uint32_t j = dep_off[i]; j < dep_off[i + 1]; ++j) {
            auto p = pos.find(deps[j]);
            if (p != pos.end() ? p->second < i : g.valid.count(deps[j]) != 0) {
                g.cons[deps[j]].push_back({h, k});
                ++cnt;
            }
        }
        g.valid.insert(h);
        g.deps[h] = cnt;
        ctx->tasks[h] = {class_id[i], priority[i], cnt == 0, false};
        made += cnt == 0 ? 1 : 0;
    }
    ctx->stats.n_groups += n;           // the host test reads the tasks pushed through the graph calls here ...
    if (n_ready) *n_ready = made;
    return HQS_OK;
}
int hqs_graph_finished(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** new_ready, uint32_t* n_new_ready) {
    GraphState& g = g_graph[ctx];
    g.new_ready.clear();
    std::vector<uint32_t> won;
    for (uint32_t i = 0; i < n; ++i)
        if (g.valid.erase(task[i])) {
            ctx->tasks[task[i]].ready = ctx->tasks[task[i]].prefilled = false;
            won.push_back(task[i]);
        }
    for (uint32_t h : won) {
        for (const auto& e : g.cons[h]) {
            const uint32_t c = e.first;
            const bool waiting = g.valid.count(c) && !ctx->tasks[c].ready && g.deps[c] > 0;
            if (g.gen[c] == e.second && waiting && --g.deps[c] == 0) {
                ctx->tasks[c].ready = true;
                g.new_ready.push_back(c);
            }
        }
        g.cons.erase(h);
    }
    std::sort(g.new_ready.begin(), g.new_ready.end());
    ctx->stats.n_levels += (uint32_t)won.size();   // ... and the tasks finished through them here
    *new_ready = g.new_ready.data();
    *n_new_ready = (uint32_t)g.new_ready.size();
    return HQS_OK;
}
}
