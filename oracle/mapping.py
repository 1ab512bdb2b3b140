"""Counts -> concrete (task, worker, variant) mapping and proactive prefilling, restated
(TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows hyperqueue/crates/tako/src/internal/scheduler/mapping.rs:
  :9-21     WorkerTaskUpdate {assigned[(task, variant)], prefills, retracts}, WorkerTaskMapping
  :23-154   create_task_mapping (take_tasks(sum), one task per worker per pass, state machine
            Waiting->Assigned / Prefilled->Retracting(+retract+redirect) / Retracting->redirect update,
            per-worker stable sort by priority descending)
  :156-230  process_proactive_filling
Where the reference iterates hash maps (arbitrary order: mapping.rs:36,42) this restatement uses
ascending (rq, variant) and ascending worker id, one admissible order; the reference's own tests
compare modulo that freedom (tests/utils/scheduler.rs:97-106 eq_class).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Tuple

from .solver import SchedulingSolution


@dataclass
class WorkerTaskUpdate:
    assigned: List[Tuple[object, int]] = field(default_factory=list)
    prefills: List[object] = field(default_factory=list)
    retracts: List[object] = field(default_factory=list)


@dataclass
class WorkerTaskMapping:
    workers: Dict[int, WorkerTaskUpdate] = field(default_factory=dict)

    def update(self, w_id: int) -> WorkerTaskUpdate:
        up = self.workers.get(w_id)
        if up is None:
            up = self.workers[w_id] = WorkerTaskUpdate()
        return up

    def n_assigned(self) -> int:
        return sum(len(u.assigned) for u in self.workers.values())


def create_task_mapping(core, solution: SchedulingSolution) -> WorkerTaskMapping:
    mapping = WorkerTaskMapping()
    redirects = core.scheduler_state.redirects
    for (rq_id, v_id) in sorted(solution.sn_counts):
        counts = dict(sorted(solution.sn_counts[(rq_id, v_id)].items()))
        rq = core.rq_map.get(rq_id).variants[v_id]
        total = sum(counts.values())
        tasks = core.task_queues.get(rq_id).take_tasks(total)
        if not tasks:
            continue
        idx = 0
        done = False
        if all(core.tasks[t].state == "waiting" for t in tasks):
            # Every task goes Waiting -> Assigned (mapping.rs:55-66): the round-robin below is then a pure assignment
            # of task ids to workers, and k insert_sn_task calls on one worker equal one remove_multiple(rq, k)
            # (workerload.rs:167-178: k saturating subtractions == one by k * amount).  Same result, without a Python
            # call per task and resource entry — the benchmark's reference arm runs this on 1 M tasks per tick.
            per_worker = {w_id: [] for w_id in counts}
            while not done:
                for w_id in counts:
                    if counts[w_id] <= 0:
                        continue
                    counts[w_id] -= 1
                    per_worker[w_id].append(tasks[idx])
                    idx += 1
                    if idx >= len(tasks):
                        done = True
                        break
            for w_id, tids in per_worker.items():
                if not tids:
                    continue
                worker = core.workers[w_id]
                worker.free.remove_multiple(rq, len(tids))
                assert worker.assigned_tasks.isdisjoint(tids)
                worker.assigned_tasks.update(tids)
                up = mapping.update(w_id).assigned
                for task_id in tids:
                    task = core.tasks[task_id]
                    task.state, task.worker, task.rv = "assigned", w_id, v_id
                    up.append((task_id, v_id))
            continue
        while not done:
            for w_id in counts:
                if counts[w_id] <= 0:
                    continue
                counts[w_id] -= 1
                task_id = tasks[idx]
                worker = core.workers[w_id]
                worker.insert_sn_task(task_id, rq)
                task = core.tasks[task_id]
                if task.state == "waiting":
                    mapping.update(w_id).assigned.append((task_id, v_id))
                    task.state, task.worker, task.rv = "assigned", w_id, v_id
                elif task.state == "retracting":
                    old_worker = task.worker
                    if old_worker != w_id:
                        prev = redirects.get(task_id)
                        redirects[task_id] = (w_id, v_id)
                        if prev is not None:
                            old_target, old_v = prev
                            core.workers[old_target].remove_sn_task(
                                task_id, core.rq_map.get(task.rq_id).variants[old_v])
                elif task.state == "prefilled":
                    old_worker = task.worker
                    core.workers[old_worker].prefilled_tasks.remove(task_id)
                    mapping.update(old_worker).retracts.append(task_id)
                    assert task_id not in redirects
                    redirects[task_id] = (w_id, v_id)
                    task.state = "retracting"          # worker stays the OLD worker
                else:
                    raise AssertionError(f"unreachable task state {task.state}")
                idx += 1
                if idx >= len(tasks):
                    done = True
                    break

    for up in mapping.workers.values():
        up.assigned.sort(key=lambda tv: -core.tasks[tv[0]].priority)     # stable, Reverse(priority)

    process_proactive_filling(core, mapping)
    return mapping


def process_proactive_filling(core, mapping: WorkerTaskMapping) -> None:
    cfg = core.scheduler_state.config
    top_priority = core.task_queues.top_priority()
    for queue in core.task_queues:
        if queue.top_priority() != top_priority:
            continue
        size = max(0, queue.top_size_no_prefill() - cfg.proactive_filling_reserve)
        if size == 0:
            continue
        eligible = []
        for w_id in sorted(core.workers):
            worker = core.workers[w_id]
            if not worker.is_sn():
                continue
            up = mapping.workers.get(w_id)
            if up is None or not any(core.tasks[t].rq_id == queue.resource_rq_id for t, _ in up.assigned):
                continue
            if any(core.tasks[t].rq_id == queue.resource_rq_id for t in worker.prefilled_tasks):
                continue
            eligible.append(worker)
        if not eligible:
            continue
        prefill_size = min(size // len(eligible), cfg.proactive_filling_max)
        if prefill_size == 0:
            continue
        for worker in eligible:
            tasks = queue.take_tasks_for_prefill(prefill_size)
            for t in tasks:
                task = core.tasks[t]
                assert task.state == "waiting"
                task.state, task.worker = "prefilled", worker.id
                worker.prefilled_tasks.add(t)
            mapping.update(worker.id).prefills.extend(tasks)
