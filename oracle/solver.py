"""The MILP scheduling solver, restated (TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows hyperqueue/crates/tako/src/internal/scheduler/solver.rs:
  :10-14    SchedulingSolution {sn_counts[(rq, variant)][worker] = u32}
  :16-62    worker list (sn-capable, sorted by id), resource_sums (MAX counts as 1.0)
  :75-174   per worker: placement variables for every feasible (batch, variant), reservation
            booleans, min-utilisation rows, per-(worker, resource) capacity rows
  :211-235  blocker indicator booleans
  :240-410  batch-size rows and priority-cut rows (with gaps)
  :412-460  solve, round, extract
  :479-518  add_min_utilization     :520-549  create_sn_var (objective coefficient)
Multi-node requests (solver.rs:81-101, 175-209, 551-575) are NOT restated (out of the first slice,
SURVEY.md §8(f) row 4): a multi-node batch raises NotImplementedError.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

from .batches import TaskBatch
from .lp import EQ, MAX, MIN, LpSolver
from .model import AMOUNT_MAX, CPU_RESOURCE_ID, as_f64


@dataclass
class SchedulingSolution:
    sn_counts: Dict[Tuple[int, int], Dict[int, int]] = field(default_factory=dict)
    objective: float = 0.0
    n_vars: int = 0
    n_rows: int = 0
    solved: bool = True


def _sn_objective(rq, n_workers: int, w_idx: int, worker, resource_sums: List[float]) -> float:
    # create_sn_var (solver.rs:520-549)
    s = 0.0
    for e in rq.entries:
        g = resource_sums[e.resource_id] if e.resource_id < len(resource_sums) else 0.0
        if g < 0.000001:
            continue
        a = e.amount_or_none_if_all()
        if a is None:
            a = worker.resources.get(e.resource_id)
        s += as_f64(a) / g
    return s * float(n_workers - w_idx) * rq.weight_f64() / float(n_workers)


def _add_min_utilization(lp: LpSolver, worker, cpu_terms: List[Tuple[int, float]]) -> None:
    # solver.rs:479-518
    if not worker.is_sn():
        return
    all_cpus_amount = worker.resources.get(CPU_RESOURCE_ID)
    if all_cpus_amount == AMOUNT_MAX:
        return
    all_cpus = as_f64(all_cpus_amount)
    free_cpus = as_f64(worker.free.get(CPU_RESOURCE_ID))
    min_cpus = all_cpus * (float(worker.min_utilization) - 1.0) + free_cpus
    if min_cpus < 0.0001:
        return
    m = lp.add_bool_variable(0.0)
    lp.add_constraint(MIN, 0.0, cpu_terms + [(m, -min_cpus)])
    lp.add_constraint(MAX, 0.0, cpu_terms + [(m, -all_cpus)])


def run_scheduling_solver(core, now: float, batches: Sequence[TaskBatch],
                          custom_workers: Optional[Sequence] = None,
                          time_limit: Optional[float] = None, mip_rel_gap: Optional[float] = None,
                          accept_incumbent: bool = False) -> SchedulingSolution:
    result = SchedulingSolution()
    if core.rq_map.is_empty():
        return result
    n_resources = core.n_resources()
    rq_map = core.rq_map
    if custom_workers is not None:
        workers = list(custom_workers)
    else:
        workers = sorted((w for w in core.workers.values() if w.is_sn()), key=lambda w: w.id)

    resource_sums = [0.0] * n_resources
    for w in workers:
        for r, c in enumerate(w.free.n[:n_resources]):
            resource_sums[r] += 1.0 if c == AMOUNT_MAX else as_f64(c)
    n_workers = len(workers)

    lp = LpSolver()
    placements: Dict[Tuple[int, int, int], int] = {}
    count_vars: Dict[int, List[int]] = {}
    # NB (reference quirk kept): the per-resource term lists persist across workers and are only
    # cleared after a row was (or could have been) emitted; a MAX free amount skips the clear
    # (solver.rs:158-172).
    res_rows: List[List[Tuple[int, float]]] = [[] for _ in range(n_resources)]

    for w_idx, w in enumerate(workers):
        cpu_terms: List[Tuple[int, float]] = []
        for b in batches:
            rqv = rq_map.get(b.resource_rq_id)
            has_variant = False
            for v_idx, rq in enumerate(rqv.variants):
                if rq.is_multi_node():
                    raise NotImplementedError("multi-node requests are not restated in the oracle")
                if (not w.is_request_blocked(b.resource_rq_id, v_idx)
                        and w.has_time_to_run(rq.min_time, now)
                        and w.have_immediate_resources_for_rq(rq)):
                    has_variant = True
                    x = lp.add_nat_variable(_sn_objective(rq, n_workers, w_idx, w, resource_sums))
                    placements[(w.id, b.resource_rq_id, v_idx)] = x
                    count_vars.setdefault(b.resource_rq_id, []).append(x)
                    for e in rq.entries:
                        a = e.amount_or_none_if_all()
                        if a is None:
                            a = w.resources.get(e.resource_id)
                        res_rows[e.resource_id].append((x, as_f64(a)))
                        if e.resource_id == CPU_RESOURCE_ID:
                            cpu_terms.append((x, as_f64(a)))
            # reservation boolean (solver.rs:133-151)
            if (not has_variant and not rqv.is_multi_node() and not b.limit_reached and b.is_blocker
                    and w.is_capable_to_run_rqv(rqv, now) and w.is_sn()):
                rv = lp.add_bool_variable(w_idx / float(n_workers * 100))
                count_vars.setdefault(b.resource_rq_id, []).append(rv)
                for r, cnt in w.free.iter_pairs():
                    res_rows[r].append((rv, as_f64(cnt)))

        if w.min_utilization > 0.001:
            _add_min_utilization(lp, w, cpu_terms)

        for r, terms in enumerate(res_rows):
            free = w.free.get(r)
            if free == AMOUNT_MAX:
                continue
            if terms:
                lp.add_constraint(MAX, as_f64(free), list(terms))
            terms.clear()

    # blocker indicators: B[(rq, s)] may be 0 only if at least s tasks of rq are scheduled
    bvars: Dict[Tuple[int, int], int] = {}

    def get_bvar(blocker_rq: int, size: int) -> int:
        key = (blocker_rq, size)
        v = bvars.get(key)
        if v is None:
            v = lp.add_bool_variable(0.0)
            # The reference unwraps count_vars[blocker] here; an empty list is the only sane
            # completion when no variable exists (forces B = 1).
            terms = [(x, 1.0) for x in count_vars.get(blocker_rq, [])]
            lp.add_constraint(MIN, float(size), terms + [(v, float(size))])
            bvars[key] = v
        return v

    capable: Dict[Tuple[int, int], bool] = {}
    for b in batches:
        counts = count_vars.get(b.resource_rq_id)
        if counts is None:
            continue
        b_rqv = rq_map.get(b.resource_rq_id)
        if not b.limit_reached:
            lp.add_constraint(MAX, float(b.size), [(x, 1.0) for x in counts])
        batch_size = float(b.size)
        blocked_by_unbounded = set()
        for cut in b.cuts:
            cut_size = float(cut.size)
            for blocker_rq, blocking_size in cut.blockers:
                zero_cond: List[int] = []
                blocker_rqv = rq_map.get(blocker_rq)
                for w in workers:
                    if not w.is_sn():
                        continue
                    ck = (w.id, blocker_rq)
                    cap = capable.get(ck)
                    if cap is None:                       # pure in (worker, blocker) within one tick
                        cap = capable[ck] = w.is_capable_to_run_rqv(blocker_rqv, now)
                    if not cap:
                        continue
                    gap = core.scheduler_state.gap_cache.get_gap(
                        blocker_rq, b.resource_rq_id, w.resources,
                        [(core.tasks[t].rq_id, core.tasks[t].rv) for t in w.assigned_tasks], rq_map)
                    xs = [placements[(w.id, b.resource_rq_id, v)] for v in range(len(b_rqv.variants))
                          if (w.id, b.resource_rq_id, v) in placements]
                    if gap > 0:
                        if blocking_size is not None:
                            bv = get_bvar(blocker_rq, blocking_size)
                            lp.add_constraint(MAX, cut_size + batch_size + float(gap),
                                              [(x, 1.0) for x in xs] + [(bv, batch_size)])
                        else:
                            lp.add_constraint(MAX, cut_size + float(gap), [(x, 1.0) for x in xs])
                    else:
                        zero_cond.extend(xs)
                if not zero_cond:
                    continue
                if blocking_size is not None:
                    bv = get_bvar(blocker_rq, blocking_size)
                    lp.add_constraint(MAX, batch_size + cut_size,
                                      [(x, 1.0) for x in zero_cond] + [(bv, batch_size)])
                elif blocker_rq not in blocked_by_unbounded:
                    blocked_by_unbounded.add(blocker_rq)
                    lp.add_constraint(MAX, cut_size, [(x, 1.0) for x in zero_cond])

    result.n_vars = len(lp.obj)
    result.n_rows = len(lp.row_lo)
    sol = lp.solve(time_limit=time_limit, mip_rel_gap=mip_rel_gap, accept_incumbent=accept_incumbent)
    core.last_solver_info = {"hit_time_limit": getattr(lp, "last_status", 0) == 1, "variables": len(lp.obj), "rows": len(lp.row_lo)}
    if sol is None:
        result.solved = False        # non-optimal => empty solution, nothing scheduled (solver.rs:412-415)
        return result
    values, result.objective = sol

    for b in batches:
        rqv = rq_map.get(b.resource_rq_id)
        for v_id in range(len(rqv.variants)):
            counts = {}
            for w in workers:
                x = placements.get((w.id, b.resource_rq_id, v_id))
                if x is None:
                    continue
                c = int(math.floor(values[x] + 0.5))
                if c > 0:
                    counts[w.id] = c
            if counts:
                result.sn_counts[(b.resource_rq_id, v_id)] = counts
    return result
