// TEST DOUBLE of hqs_graph_cancel (include/hqsched.h) — test infrastructure, never shipped or loaded by the product.  It is
// fake_hqsched_graph.cpp (compiled into this translation unit, so that the call reaches its graph state) plus the cancel in
// host memory: every named VALID handle leaves, and so does, transitively, every consumer still waiting on the incarnation
// its edge was made for; the handles that left come back ascending.
#include "fake_hqsched_graph.cpp"

namespace {
std::map<const hqs_ctx*, std::vector<uint32_t>> g_cancelled;
}

extern "C" int hqs_graph_cancel(hqs_ctx* ctx, uint32_t n, const uint32_t* task, const uint32_t** cancelled, uint32_t* n_cancelled) {
    GraphState& g = g_graph[ctx];
    std::vector<uint32_t>& out = g_cancelled[ctx];
    out.clear();
    std::set<uint32_t> gone;
    std::vector<uint32_t> stack;
    for (uint32_t i = 0; i < n; ++i)
        if (g.valid.count(task[i]) && gone.insert(task[i]).second) stack.push_back(task[i]);
    while (!stack.empty()) {
        const uint32_t h = stack.back();
        stack.pop_back();
        for (const auto& e : g.cons[h]) {
            const uint32_t c = e.first;
            const bool waiting = g.valid.count(c) && !ctx->tasks[c].ready && g.deps[c] > 0;
            if (g.gen[c] == e.second && waiting && gone.insert(c).second) stack.push_back(c);
        }
    }
    for (uint32_t h : gone) {
        g.valid.erase(h);
        g.cons.erase(h);
        ctx->tasks[h].ready = ctx->tasks[h].prefilled = false;
        out.push_back(h);
    }
    *cancelled = out.data();
    *n_cancelled = (uint32_t)out.size();
    return HQS_OK;
}
