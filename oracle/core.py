"""Server core state and the tick driver, restated (TEST INFRASTRUCTURE — see oracle/__init__.py).

Follows (paths relative to hyperqueue/crates/tako/src/internal/):
  server/core.rs:41-62 (Core), :207-235 (add_task / remove_task)
  server/task.rs:22-43,115-125,175-177     Task, TaskRuntimeState, priority()
  server/reactor.rs:188-220                on_new_tasks (dependency counting, ready insertion)
  server/reactor.rs:500-580                task_finished (resource return, readiness propagation)
  scheduler/state.rs:4-28                  SchedulerConfig (reserve 16 / max 40), SchedulerState
  scheduler/main.rs:40-46                  run_scheduling_inner = batches -> solver -> mapping
  tests/utils/env.rs:31-261                TestEnv helpers (worker ids start at 50, task ids at 1)
Only the parts of the reactor that feed the single-node tick are restated; retract responses, worker
loss, multi-node tasks and the RPC layer are out of scope (SURVEY.md §8).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

from .batches import create_task_batches
from .gap import GapCache
from .mapping import WorkerTaskMapping, create_task_mapping
from .model import (ResourceRequestVariants, ResourceRqMap, Worker, WorkerResources,
                    priority_from_user)
from .solver import run_scheduling_solver
from .taskqueue import TaskQueues


@dataclass
class SchedulerConfig:
    proactive_filling_reserve: int = 16      # state.rs:14-21
    proactive_filling_max: int = 40


@dataclass
class SchedulerState:
    gap_cache: GapCache = field(default_factory=GapCache)
    config: SchedulerConfig = field(default_factory=SchedulerConfig)
    redirects: Dict[object, Tuple[int, int]] = field(default_factory=dict)


@dataclass
class Task:
    id: object
    rq_id: int
    user_priority: int = 0
    state: str = "waiting"        # waiting | assigned | running | prefilled | retracting | finished
    unfinished_deps: int = 0
    worker: Optional[int] = None
    rv: Optional[int] = None
    deps: Tuple = ()
    consumers: List = field(default_factory=list)

    @property
    def priority(self) -> int:
        return priority_from_user(self.user_priority)     # task.rs:175-177

    def is_ready(self) -> bool:
        return self.state == "waiting" and self.unfinished_deps == 0

    def is_assigned(self) -> bool:
        return self.state == "assigned"


class Core:
    def __init__(self) -> None:
        self.tasks: Dict[object, Task] = {}
        self.workers: Dict[int, Worker] = {}
        self.task_queues = TaskQueues()
        self.rq_map = ResourceRqMap()
        self.scheduler_state = SchedulerState()
        self.resource_names: List[str] = ["cpus"]        # map.rs:7-31: cpus is always id 0

    # resources / classes -------------------------------------------------------------------
    def get_or_create_resource_id(self, name: str) -> int:
        if name not in self.resource_names:
            self.resource_names.append(name)
        return self.resource_names.index(name)

    def n_resources(self) -> int:
        return len(self.resource_names)

    def get_or_create_resource_rq_id(self, rqv: ResourceRequestVariants) -> int:
        # reactor.rs get_or_create_raw_resource_rq_id: a new class gets a new TaskQueue
        rq_id, is_new = self.rq_map.get_or_create(rqv)
        if is_new:
            self.task_queues.add_task_queue()
        return rq_id

    # workers --------------------------------------------------------------------------------
    def new_worker(self, worker: Worker) -> None:
        # reactor.rs:20-32 on_new_worker (only the state change)
        assert worker.id not in self.workers
        self.workers[worker.id] = worker

    # tasks ----------------------------------------------------------------------------------
    def on_new_tasks(self, tasks: Iterable[Task]) -> List:
        retracted: List = []
        for task in tasks:
            count = 0
            kept = []
            for d in task.deps:
                dep = self.tasks.get(d)
                if dep is not None:
                    dep.consumers.append(task.id)
                    if dep.state != "finished":
                        count += 1
                    kept.append(d)
            task.deps = tuple(kept)
            task.unfinished_deps = count
            task.state = "waiting"
            if task.is_ready():
                self.task_queues.add_ready_task(task.id, task.rq_id, task.priority, retracted)
            assert task.id not in self.tasks
            self.tasks[task.id] = task
        self._process_retracted(retracted)
        return retracted

    def _process_retracted(self, retracted: List) -> None:
        # reactor.rs:34-62 process_retracted: a disposed prefill goes back to Waiting on the server
        # side (the RetractTasks message itself is out of scope here).
        for t in retracted:
            task = self.tasks[t]
            if task.state == "prefilled":
                self.workers[task.worker].prefilled_tasks.discard(t)
                task.state, task.worker = "waiting", None

    def remove_from_ready_queue(self, task_id) -> None:
        task = self.tasks[task_id]
        self.task_queues.get(task.rq_id).remove(task_id, task.priority)

    def assign_task(self, task_id, worker_id: int, rv: int = 0) -> None:
        """TestEnv::assign_task (tests/utils/env.rs:176-207)."""
        task = self.tasks[task_id]
        assert task.is_ready(), f"task {task_id} is not ready"
        self.remove_from_ready_queue(task_id)
        task.state, task.worker, task.rv = "assigned", worker_id, rv
        self.workers[worker_id].insert_sn_task(task_id, self.rq_map.get(task.rq_id).variants[rv])

    def start_task(self, task_id, rv: int = 0) -> None:
        """on_task_update(Running) for an Assigned task (reactor.rs:263-345), same variant only."""
        task = self.tasks[task_id]
        assert task.state == "assigned"
        task.state = "running"

    def task_finished(self, worker_id: int, task_id) -> bool:
        task = self.tasks.get(task_id)
        if task is None:
            return False
        if task.state in ("assigned", "running"):
            assert task.worker == worker_id
            self.workers[worker_id].remove_sn_task(task_id, self.rq_map.get(task.rq_id).variants[task.rv])
        else:
            raise AssertionError(f"task_finished in state {task.state} is not restated")
        task.state = "finished"
        retracted: List = []
        for c in task.consumers:
            t = self.tasks[c]
            t.unfinished_deps -= 1
            if t.unfinished_deps == 0:
                self.task_queues.add_ready_task(t.id, t.rq_id, t.priority, retracted)
        self._process_retracted(retracted)
        del self.tasks[task_id]
        return True

    # the tick ---------------------------------------------------------------------------------
    def schedule_mapping(self, now: float = 0.0, time_limit: Optional[float] = None,
                         mip_rel_gap: Optional[float] = None, accept_incumbent: bool = False) -> WorkerTaskMapping:
        """run_scheduling_inner minus send_messages (main.rs:40-46, env.rs:257-261)."""
        batches = create_task_batches(self, now)
        solution = run_scheduling_solver(self, now, batches, time_limit=time_limit, mip_rel_gap=mip_rel_gap,
                                         accept_incumbent=accept_incumbent)
        self.last_solution = solution
        return create_task_mapping(self, solution)

    # invariants -------------------------------------------------------------------------------
    def sanity_check(self) -> None:
        """Worker half of Core::sanity_check (server/worker.rs:236-271): replay every assigned task
        against the worker's totals and compare with the tracked free vector."""
        for w in self.workers.values():
            res = w.resources.clone()
            for t in w.assigned_tasks:
                task = self.tasks[t]
                if task.state in ("assigned", "running"):
                    wid, rv = task.worker, task.rv
                elif task.state == "retracting":
                    wid, rv = self.scheduler_state.redirects[t]
                else:
                    raise AssertionError(f"invalid state {task.state}")
                assert wid == w.id
                rq = self.rq_map.get(task.rq_id).variants[rv]
                assert res.is_capable_to_run_request(rq)
                res.remove(rq)
            assert w.free.n[:len(res.n)] == res.n or _trim(w.free.n) == _trim(res.n), (w.id, w.free, res)
            for t in w.prefilled_tasks:
                task = self.tasks[t]
                assert task.state == "prefilled" and task.worker == w.id


def _trim(v: Sequence[int]) -> List[int]:
    v = list(v)
    while v and v[-1] == 0:
        v.pop()
    return v
