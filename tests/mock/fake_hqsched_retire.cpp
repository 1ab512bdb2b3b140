// TEST DOUBLE of hqs_handles_compact (include/hqsched.h) — test infrastructure, never shipped or loaded by the product.  It
// is fake_hqsched_graph_cancel.cpp (compiled into this translation unit, so that the call reaches its ready set and graph
// state) plus the renumbering in host memory: the survivors are the VALID handles and the named ones; survivor i in ascending
// old handle becomes handle i with its task, dependency count, incarnation and consumer list; an edge whose consumer no
// longer waits on the edge's incarnation is dropped; the old handles come back ascending.
#include "fake_hqsched_graph_cancel.cpp"

namespace {
std::map<const hqs_ctx*, std::vector<uint32_t>> g_old_of_new;
}

extern "C" int hqs_handles_compact(hqs_ctx* ctx, uint32_t n_keep, const uint32_t* keep, const uint32_t** old_of_new,
                                   uint32_t* n_kept) {
    GraphState& g = g_graph[ctx];
    hqs_stats st;
    hqs_get_stats(ctx, &st);
    for (uint32_t i = 0; i < n_keep; ++i)
        if (keep[i] >= st.n_handles) { ctx->err = "keep handle out of range"; return HQS_E_INVALID; }
    std::set<uint32_t> kept(g.valid.begin(), g.valid.end());
    kept.insert(keep, keep + n_keep);
    std::vector<uint32_t>& order = g_old_of_new[ctx];
    order.assign(kept.begin(), kept.end());
    std::map<uint32_t, uint32_t> new_of;
    for (uint32_t i = 0; i < order.size(); ++i) new_of[order[i]] = i;
    GraphState ng;
    std::map<uint32_t, hqs_ctx::T> tasks;
    for (uint32_t i = 0; i < order.size(); ++i) {
        const uint32_t o = order[i];
        if (ctx->tasks.count(o)) tasks[i] = ctx->tasks[o];
        if (g.valid.count(o)) ng.valid.insert(i);
        if (g.deps.count(o)) ng.deps[i] = g.deps[o];
        if (g.gen.count(o)) ng.gen[i] = g.gen[o];
    }
    for (const auto& kv : g.cons) {
        for (const auto& e : kv.second) {
            const uint32_t c = e.first;
            const bool waits = g.valid.count(c) && !ctx->tasks[c].ready && g.deps[c] > 0 && g.gen[c] == e.second;
            if (waits) ng.cons[new_of.at(kv.first)].push_back({new_of.at(c), e.second});
        }
    }
    ng.new_ready = g.new_ready;
    g = ng;
    ctx->tasks.swap(tasks);
    *old_of_new = order.data();
    *n_kept = (uint32_t)order.size();
    return HQS_OK;
}
