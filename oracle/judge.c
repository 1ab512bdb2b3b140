/* Plain-C restatement of the per-(worker, class, variant) admission predicate and the per-(worker,
 * resource) capacity check (TEST INFRASTRUCTURE — see oracle/__init__.py and oracle/judge.py).
 *
 * Follows hyperqueue/crates/tako/src/internal/
 *   scheduler/solver.rs:103-105      !blocked && has_time_to_run && have_immediate_resources_for_rq
 *   server/workerload.rs:77-83       is_capable_to_run_request: every entry's min_amount <= free
 *   common/resources/request.rs:34-36  min_amount of `All` is one fraction
 *   scheduler/solver.rs:120-124,158-173  capacity row: sum(cap * x) <= free, cap = total for `All`
 * Used by the tests to cross-check oracle/judge.py on large assignment lists.
 *
 * Returns the number of violations found (0 = every assignment feasible).
 */
#include <stdint.h>
#include <stdlib.h>

#define AMOUNT_MAX (~(uint64_t)0)

int64_t hq_judge(uint32_t W, uint32_t R, uint32_t Q, uint32_t V,
                 const uint64_t *class_amounts /* [Q][V][R] */, const uint8_t *class_all /* [Q][V][R] */,
                 const uint64_t *class_min_time_ms /* [Q][V] */, const uint64_t *free_rw /* [W][R] */,
                 const uint64_t *total_rw /* [W][R] */, const uint64_t *remaining_time_ms /* [W] */,
                 const uint8_t *blocked /* [W][Q][V] or NULL */, const uint32_t *task_class,
                 uint64_t n, const uint32_t *a_task, const uint16_t *a_worker, const uint8_t *a_variant)
{
    int64_t violations = 0;
    uint64_t *counts = calloc((size_t)W * Q * V, sizeof(uint64_t));
    if (!counts) return -1;
    for (uint64_t i = 0; i < n; ++i) {
        uint32_t w = a_worker[i], c = task_class[a_task[i]], v = a_variant[i];
        if (w >= W || c >= Q || v >= V) { violations++; continue; }
        counts[((size_t)w * Q + c) * V + v]++;
    }
    for (uint32_t w = 0; w < W; ++w) {
        for (uint32_t r = 0; r < R; ++r) {
            /* 128-bit accumulator: no overflow however large the amounts are */
            unsigned __int128 used = 0;
            for (uint32_t c = 0; c < Q; ++c)
                for (uint32_t v = 0; v < V; ++v) {
                    uint64_t k = counts[((size_t)w * Q + c) * V + v];
                    if (!k) continue;
                    size_t e = (((size_t)c * V) + v) * R + r;
                    uint64_t cap = class_all[e] ? total_rw[(size_t)w * R + r] : class_amounts[e];
                    used += (unsigned __int128)cap * k;
                    if (r == 0) { /* admission predicate, once per (w, c, v) */
                        if (blocked && blocked[((size_t)w * Q + c) * V + v]) violations++;
                        if (remaining_time_ms[w] != AMOUNT_MAX &&
                            class_min_time_ms[(size_t)c * V + v] > remaining_time_ms[w]) violations++;
                        for (uint32_t r2 = 0; r2 < R; ++r2) {
                            size_t e2 = (((size_t)c * V) + v) * R + r2;
                            uint64_t need = class_all[e2] ? 1 : class_amounts[e2];
                            if (need && need > free_rw[(size_t)w * R + r2]) violations++;
                        }
                    }
                }
            if (free_rw[(size_t)w * R + r] != AMOUNT_MAX && used > free_rw[(size_t)w * R + r]) violations++;
        }
    }
    free(counts);
    return violations;
}
