"""Stand-alone feasibility judge (TEST INFRASTRUCTURE — see oracle/__init__.py).

"Every emitted assignment must be bit-exact feasible against the reference's own ResourceRequest
check": this module restates exactly that check, independent of any scheduler:

  per (worker, class, variant)   the solver's admission predicate
      !is_request_blocked && has_time_to_run && have_immediate_resources_for_rq
      (hyperqueue/crates/tako/src/internal/scheduler/solver.rs:103-105,
       server/worker.rs:273-278,320-326,328-334, server/workerload.rs:77-83;
       `All` needs 1 fraction: common/resources/request.rs:34-36)
  per (worker, resource)         the capacity row  sum cap * x <= free   with cap = amount, or the
      worker's TOTAL for `All` (solver.rs:120-124,158-173); a MAX free amount has no row
  replay                          Worker::sanity_check (server/worker.rs:236-271): removing the
      tasks one by one never needs more than what is left

Amounts are exact integers (Python ints: no u64 overflow in the sums).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

AMOUNT_MAX = (1 << 64) - 1
TIME_INF = (1 << 64) - 1


class JudgeResult:
    def __init__(self) -> None:
        self.n = 0
        self.violations: List[str] = []

    @property
    def ok(self) -> bool:
        return not self.violations

    def __repr__(self) -> str:
        return f"JudgeResult(n={self.n}, ok={self.ok}, first={self.violations[:3]})"


def judge_assignments(class_amounts: np.ndarray, class_all: np.ndarray, class_nvar: np.ndarray,
                      class_min_time_ms: np.ndarray, free: np.ndarray, total: np.ndarray,
                      remaining_time_ms: np.ndarray, blocked: Optional[np.ndarray],
                      task_class: np.ndarray, a_task: np.ndarray, a_worker: np.ndarray, a_variant: np.ndarray,
                      ready_mask: Optional[np.ndarray] = None, max_report: int = 10) -> JudgeResult:
    """class_amounts [Q][V][R] u64, class_all [Q][V][R] bool, class_nvar [Q], class_min_time_ms [Q][V],
    free/total [W][R] u64 (tick start), remaining_time_ms [W] (TIME_INF = none),
    blocked [W][Q][V] bool or None, task_class [H]; assignment triples a_* (worker = index)."""
    res = JudgeResult()
    n = int(a_task.shape[0])
    res.n = n
    W, R = free.shape
    Q, V = class_amounts.shape[:2]

    def bad(msg: str) -> None:
        if len(res.violations) < max_report:
            res.violations.append(msg)

    if n == 0:
        return res
    a_task = a_task.astype(np.int64); a_worker = a_worker.astype(np.int64); a_variant = a_variant.astype(np.int64)
    if np.unique(a_task).shape[0] != n:
        bad("a task was assigned more than once")
    if a_worker.max() >= W:
        bad("worker index out of range"); return res
    if ready_mask is not None and not ready_mask[a_task].all():
        bad("a task that was not ready was assigned")
    cls = task_class[a_task].astype(np.int64)
    if (a_variant >= class_nvar[cls]).any():
        bad("variant index out of range"); return res

    # counts[w][c][v]
    counts = np.zeros((W, Q, V), dtype=np.int64)
    np.add.at(counts, (a_worker, cls, a_variant), 1)
    ws, cs, vs = np.nonzero(counts)
    for w, c, v in zip(ws.tolist(), cs.tolist(), vs.tolist()):
        # admission predicate at tick start
        if blocked is not None and blocked[w, c, v]:
            bad(f"worker {w}: class {c} variant {v} is blocked")
        rt = int(remaining_time_ms[w])
        if rt != TIME_INF and int(class_min_time_ms[c, v]) > rt:
            bad(f"worker {w}: class {c} variant {v} needs {int(class_min_time_ms[c, v])} ms, {rt} ms left")
        for r in range(R):
            need = 1 if class_all[c, v, r] else int(class_amounts[c, v, r])
            if need and need > int(free[w, r]):
                bad(f"worker {w}: class {c} variant {v} needs {need} of resource {r}, {int(free[w, r])} free")
    # capacity rows
    for w in range(W):
        cw = counts[w]
        if not cw.any():
            continue
        for r in range(R):
            if int(free[w, r]) == AMOUNT_MAX:
                continue
            used = 0
            cs2, vs2 = np.nonzero(cw)
            for c, v in zip(cs2.tolist(), vs2.tolist()):
                cap = int(total[w, r]) if class_all[c, v, r] else int(class_amounts[c, v, r])
                used += cap * int(cw[c, v])
            if used > int(free[w, r]):
                bad(f"worker {w}: resource {r} over-committed: {used} > {int(free[w, r])}")
    return res


def replay_free_after(class_amounts: np.ndarray, class_all: np.ndarray, free: np.ndarray, total: np.ndarray,
                      task_class: np.ndarray, a_task: np.ndarray, a_worker: np.ndarray,
                      a_variant: np.ndarray) -> np.ndarray:
    """WorkerResources::remove for every assignment (workerload.rs:156-165): the free vectors the
    reference would hold after create_task_mapping.  Exact (object ints), saturating at zero."""
    W, R = free.shape
    out = [[int(free[w, r]) for r in range(R)] for w in range(W)]
    Q, V = class_amounts.shape[:2]
    counts = np.zeros((W, Q, V), dtype=np.int64)
    if a_task.shape[0]:
        np.add.at(counts, (a_worker.astype(np.int64), task_class[a_task.astype(np.int64)].astype(np.int64),
                           a_variant.astype(np.int64)), 1)
    ws, cs, vs = np.nonzero(counts)
    for w, c, v in zip(ws.tolist(), cs.tolist(), vs.tolist()):
        k = int(counts[w, c, v])
        for r in range(R):
            if class_all[c, v, r]:
                out[w][r] = 0
            elif class_amounts[c, v, r] and out[w][r] != AMOUNT_MAX:
                out[w][r] = max(0, out[w][r] - int(class_amounts[c, v, r]) * k)
    return np.array(out, dtype=np.uint64)
